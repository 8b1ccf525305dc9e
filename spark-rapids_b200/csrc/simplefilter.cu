// simplefilter.cu — fast path of GpuFilter's selection vector (basicPhysicalOperators.scala:1148-1224) for the commonest
// predicate shape: a conjunction of comparisons between NOT NULL fixed-width integer columns (ints, dates, timestamps,
// DECIMAL32/64) and literals — date ranges, key bounds, flags (TPC-H q3: o_orderdate < d, l_shipdate > d; q6's five terms).
// The general path interprets the predicate in the expression VM (vm.cuh) one 4096-row tile at a time; here the compiled
// program is pattern-matched on the host and a specialised kernel streams the columns with 16-byte loads (consecutive lanes
// on consecutive vectors), keeps the tile's result as a bit mask in shared memory and writes the selected row ids in order,
// coalesced, through a shared-memory stage (single pass: block scan + decoupled look-back across tiles).  Anything that does not match the shape returns false and takes the VM.
#include "prim.cuh"
#include "vm.cuh"
#include "simplefilter.cuh"

namespace b2 {

constexpr int SF_WARPS = SF_NT / 32, SF_TILE = 32768, SF_WORDS = SF_TILE / 32, SF_WWORDS = SF_WORDS / SF_WARPS;
struct SimpleWork { unsigned long long tile_counter, total; };

constexpr uint64_t SLB_AGG = 1ull << 62, SLB_PREFIX = 2ull << 62, SLB_MASK = (1ull << 62) - 1;
__device__ __forceinline__ uint64_t sf_ld(const uint64_t* p) { uint64_t v; asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void sf_st(uint64_t* p, uint64_t v) { asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

// Decoupled look-back over the per-tile counts, by the WHOLE CTA: 256 predecessors are inspected per step.  The tiles of a
// launch are uniform, so they finish counting at about the same time and nobody's prefix is ready: a warp-wide window
// (32 per step, scan.cu) made every tile walk ~all running tiles one L2 round trip at a time; this walks them 256 at a time.
// Called by every thread; returns the exclusive prefix of `tile` and publishes its inclusive prefix.
__device__ __forceinline__ int64_t sf_block_lookback(uint64_t* status, int64_t tile, uint32_t count, int64_t* s_sum, int* s_has) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (tile == 0) { if (threadIdx.x == 0) { __threadfence(); sf_st(&status[0], SLB_PREFIX | count); } return 0; }
  if (threadIdx.x == 0) { __threadfence(); sf_st(&status[tile], SLB_AGG | count); }
  int64_t excl = 0, look = tile - 1;
  while (true) {
    const int64_t idx = look - threadIdx.x;
    uint64_t v;
    if (idx >= 0) { do { v = sf_ld(&status[idx]); } while ((v >> 62) == 0); } else v = SLB_PREFIX;
    const uint32_t is_prefix = __ballot_sync(0xffffffffu, (v >> 62) == 2);
    const int first = is_prefix ? __ffs(is_prefix) - 1 : 32;
    int64_t contrib = (lane <= first) ? (int64_t)(v & SLB_MASK) : 0;
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
    if (lane == 0) { s_sum[warp] = contrib; s_has[warp] = is_prefix != 0; }
    __syncthreads();
    bool done = false;
    for (int w = 0; w < SF_WARPS && !done; w++) { excl += s_sum[w]; done = s_has[w] != 0; }   // warp 0 holds the nearest predecessors
    __syncthreads();
    if (done) break;
    look -= SF_NT;
  }
  if (threadIdx.x == 0) { __threadfence(); sf_st(&status[tile], SLB_PREFIX | (uint64_t)(excl + count)); }
  return excl;
}

__global__ void __launch_bounds__(SF_NT) simple_filter_ids_kernel(const __grid_constant__ SimplePred sp, int64_t n, int32_t* __restrict__ ids,
                                                                  uint64_t* __restrict__ status, SimpleWork* __restrict__ work) {
  __shared__ uint32_t s_mask[SF_WORDS];              // bit r: row r of the tile passes every term
  __shared__ int32_t s_stage[SF_WARPS][1024];        // per warp: the selected ids of 1024 rows, then written out coalesced
  __shared__ uint32_t s_wtot[SF_WARPS];
  __shared__ int64_t s_tile, s_sum[SF_WARPS];
  __shared__ int s_has[SF_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ntiles = (n + SF_TILE - 1) / SF_TILE;
  while (true) {
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(&work->tile_counter, 1ull);   // tiles in launch order: look-back never waits on an unstarted tile
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    const int64_t tile_row0 = tile * SF_TILE;
    const int tile_n = (int)min((int64_t)SF_TILE, n - tile_row0);
    sf_tile(sp, tile_row0, tile_n, s_mask, SF_WORDS);
    // warp w owns mask words [w * 128, (w + 1) * 128) = rows [w * 4096, (w + 1) * 4096) of the tile
    {
      uint32_t c = 0;
#pragma unroll
      for (int i = 0; i < SF_WWORDS / 32; i++) c += __popc(s_mask[warp * SF_WWORDS + i * 32 + lane]);
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) s_wtot[warp] = c;
    }
    __syncthreads();
    uint32_t total = 0, before = 0;
#pragma unroll
    for (int w = 0; w < SF_WARPS; w++) { if (w < warp) before += s_wtot[w]; total += s_wtot[w]; }
    const int64_t excl = sf_block_lookback(status, tile, total, s_sum, s_has);
    if (threadIdx.x == 0 && tile == ntiles - 1) work->total = (unsigned long long)(excl + total);
    // ids of the warp's rows, 1024 rows at a time: positions by a warp scan of the word popcounts, staged in shared memory,
    // written out with consecutive lanes on consecutive ids (no block barrier in this phase)
    int64_t out = excl + before;
    for (int r = 0; r < SF_WWORDS / 32; r++) {
      const int word = warp * SF_WWORDS + r * 32 + lane;
      const uint32_t m = s_mask[word];
      const uint32_t cnt = __popc(m);
      uint32_t inc = cnt;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
      const uint32_t rtot = __shfl_sync(0xffffffffu, inc, 31);
      uint32_t pos = inc - cnt;
      const int32_t r0 = (int32_t)(tile_row0 + (int64_t)word * 32);
      for (uint32_t mm = m; mm; mm &= mm - 1) s_stage[warp][pos++] = r0 + (__ffs(mm) - 1);
      __syncwarp();
      for (uint32_t i = lane; i < rtot; i += 32) ids[out + i] = s_stage[warp][i];
      out += rtot;
      __syncwarp();
    }
    __syncthreads();   // s_mask / s_wtot / s_tile are rewritten by the next tile
  }
}

// pattern match: output 0 = c0 AND c1 AND ... with c_i = (NOT NULL fixed-width integer column) <cmp> (non-null literal)
bool simple_pred_of(const Program* prog, const Table* t, SimplePred& sp) {
  memset(&sp, 0, sizeof(sp));
  const int n = prog->hdr.ninstr;
  if (prog->hdr.nouts != 1 || n < 1 || n > SF_MAX_TERMS || (int)prog->code.size() != n) return false;
  static const int truth_of[6] = {2, 5, 1, 3, 4, 6};   // EQ NE LT LE GT GE over {<, ==, >}
  int prev_dst = -1;
  for (int i = 0; i < n; i++) {
    const VMInstr& ins = prog->code[i];
    int truth;
    if (i == 0) { if (ins.op < V_EQ || ins.op > V_GE || ins.dst_nullable) return false; truth = truth_of[ins.op - V_EQ]; }
    else { if (ins.op != V_ANDCMP || ins.c.kind != OK_REG || ins.c.idx != prev_dst) return false; truth = ins.aux; }
    if (ins.mt != MT_I8 && ins.mt != MT_I16 && ins.mt != MT_I32 && ins.mt != MT_I64) return false;
    if (ins.a.kind != OK_COL || ins.b.kind != OK_LIT || ins.b.lit_null) return false;
    if (ins.a.idx < 0 || ins.a.idx >= (int)t->cols.size()) return false;
    const Column* c = t->cols[ins.a.idx];
    if (c->nullable() || c->dtype == B2_STRING || c->dtype == B2_BOOL8 || is_float(c->dtype) || dtype_width(c->dtype) != mt_width(ins.mt)) return false;
    if ((uintptr_t)c->data.p & 15) return false;   // 16-byte vector loads
    sp.t[i].col = c->data.p; sp.t[i].width = mt_width(ins.mt); sp.t[i].truth = truth;
    // literals are stored sign-extended to 64 bits (b2_expr_literal); narrower machine types compare on their own width
    int64_t lit = ins.b.lo;
    switch (ins.mt) { case MT_I8: lit = (int8_t)lit; break; case MT_I16: lit = (int16_t)lit; break; case MT_I32: lit = (int32_t)lit; break; default: break; }
    sp.t[i].lit = lit;
    prev_dst = ins.dst;
  }
  const VMOperand& out = prog->hdr.outs[0];
  if (out.kind != OK_REG || out.idx != prev_dst) return false;
  sp.n = n;
  return true;
}

// the selection vector of `prog` over `t` through the specialised kernel; false = the predicate is not of the simple shape
bool simple_filter_row_ids(const Program* prog, const Table* t, Column** out) {
  if (getenv("B2_FILTER_NO_SIMPLE")) return false;
  SimplePred sp;
  const int64_t n = t->rows;
  if (n < (1 << 16) || !simple_pred_of(prog, t, sp)) return false;
  ColGuard ids(new_column(B2_INT32, 0, n, false));
  const int64_t ntiles = (n + SF_TILE - 1) / SF_TILE;
  DevBuf work(sizeof(SimpleWork)), status((size_t)ntiles * 8);
  CUDA_CHECK(cudaMemsetAsync(work.p, 0, sizeof(SimpleWork), stream()));
  CUDA_CHECK(cudaMemsetAsync(status.p, 0, (size_t)ntiles * 8, stream()));
  const int grid = (int)std::min<int64_t>(ntiles, (int64_t)sm_count() * 5);
  launch("simple_filter_ids_kernel", simple_filter_ids_kernel, grid, SF_NT, 0, stream(), sp, n, ids.c->data.as<int32_t>(), status.as<uint64_t>(),
         work.as<SimpleWork>());
  SimpleWork hw;
  d2h(&hw, work.p, 1);
  sync();
  ids.c->size = (int64_t)hw.total;
  *out = ids.release();
  return true;
}

}  // namespace b2
