// simplefilter.cuh — the "simple predicate" shape shared by the selection-vector kernel (simplefilter.cu) and the fused
// filter + probe kernel (join.cu): a conjunction of comparisons between NOT NULL fixed-width integer columns and literals.
#pragma once
#include <cstdint>
namespace b2 {
struct Program;
struct Table;
constexpr int SF_MAX_TERMS = 8;
struct SimpleTerm { const void* col; int32_t width; int32_t truth; int64_t lit; };   // truth: bit0 '<', bit1 '==', bit2 '>'
struct SimplePred { int32_t n; int32_t pad; SimpleTerm t[SF_MAX_TERMS]; };
// pattern match of a compiled predicate program against a batch; false = not of the simple shape (the VM evaluates it)
bool simple_pred_of(const Program* prog, const Table* t, SimplePred& sp);

constexpr int SF_NT = 256;   // threads per CTA of every kernel that calls sf_term / sf_tile

#ifdef __CUDACC__
// One term over one tile: every thread tests 16-byte vectors of the column, consecutive lanes on consecutive vectors (each
// warp load covers 512 contiguous bytes; no barrier inside, 4 loads in flight per thread), and clears the bits of the failing
// rows in the tile's shared bit mask.  tile_row0 is a multiple of 16 rows, so every vector is 16-byte aligned (simple_pred_of
// checks the column's base).
template <typename T>
__device__ __forceinline__ void sf_term(const SimpleTerm& t, int64_t tile_row0, int tile_n, uint32_t* s_mask) {
  constexpr int PER = 16 / (int)sizeof(T);                 // rows per vector
  const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(t.col) + tile_row0);
  const int nvec = (tile_n + PER - 1) / PER;               // columns are padded to 64 B: a partial last vector is readable, its extra bits are already 0 in the mask
  const T lit = (T)t.lit;
#pragma unroll 4
  for (int v = threadIdx.x; v < nvec; v += SF_NT) {
    const uint4 w = __ldg(p + v);
    const T* e = reinterpret_cast<const T*>(&w);
    uint32_t pass = 0;
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int c = e[k] < lit ? 1 : (e[k] == lit ? 2 : 4);
      pass |= (uint32_t)((t.truth & c) != 0) << k;
    }
    const uint32_t fail = ~pass & ((1u << PER) - 1u);
    const int r0 = v * PER;
    if (fail) atomicAnd(&s_mask[r0 >> 5], ~(fail << (r0 & 31)));
  }
}

// The whole predicate over one tile of `tile_n` rows: the `words` words of s_mask end with bit r set iff row r of the tile
// passes every term (bits past tile_n are 0).  Called by all SF_NT threads; ends with a barrier.
__device__ __forceinline__ void sf_tile(const SimplePred& sp, int64_t tile_row0, int tile_n, uint32_t* s_mask, int words) {
  for (int i = threadIdx.x; i < words; i += SF_NT) {
    const int lo = i * 32;
    s_mask[i] = tile_n >= lo + 32 ? 0xffffffffu : (tile_n > lo ? (1u << (tile_n - lo)) - 1u : 0u);
  }
  __syncthreads();
  for (int k = 0; k < sp.n; k++) {
    const SimpleTerm& t = sp.t[k];
    switch (t.width) {
      case 1: sf_term<int8_t>(t, tile_row0, tile_n, s_mask); break;
      case 2: sf_term<int16_t>(t, tile_row0, tile_n, s_mask); break;
      case 4: sf_term<int32_t>(t, tile_row0, tile_n, s_mask); break;
      default: sf_term<int64_t>(t, tile_row0, tile_n, s_mask); break;
    }
  }
  __syncthreads();
}
#endif
}  // namespace b2
