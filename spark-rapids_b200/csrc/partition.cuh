// partition.cuh — the pieces of the stable tile-histogram partition that more than one kernel uses: the per-tile histogram
// (hash.cu's Table.partition and radix group-by passes, agg.cu's fused materialise + first pass) and the copy-out of a tile
// that has been staged in shared memory in partition order.
#pragma once
#include "common.cuh"
#include "pack16.cuh"

namespace b2 {

constexpr int PT_NT = 256, PT_STEPS = 16, PT_TILE = PT_NT * PT_STEPS, PT_MAXP = 1024;   // PT_MAXC, ScatterCols: prim.cuh
constexpr int PS_WARPS = PT_NT / 32;

#ifdef __CUDACC__
// tile_cnt[p * ntiles + tile] = rows of tile `tile` (PT_NT * STEPS rows) whose partition is p
template <typename Pid, int STEPS = PT_STEPS>
__global__ void __launch_bounds__(PT_NT) part_tile_hist_kernel(const Pid pids, int64_t n, int32_t nparts, int64_t ntiles,
                                                               int32_t* __restrict__ tile_cnt) {
  __shared__ int32_t h[PT_MAXP];
  for (int p = threadIdx.x; p < nparts; p += PT_NT) h[p] = 0;
  __syncthreads();
  const int64_t tile = blockIdx.x;
  for (int j = 0; j < STEPS; j++) {
    const int64_t i = tile * (PT_NT * STEPS) + (int64_t)j * PT_NT + threadIdx.x;
    if (i < n) { const int32_t p = pids(i); if ((uint32_t)p < (uint32_t)nparts) atomicAdd(&h[p], 1); }
  }
  __syncthreads();
  for (int p = threadIdx.x; p < nparts; p += PT_NT) tile_cnt[(int64_t)p * ntiles + tile] = h[p];
}

// Copy-out of one tile of TILE rows whose `tile_n` elements sit in `stage` in partition order: element k belongs to partition
// s_owner[k], whose run occupies stage [s_start[p], s_start[p + 1]) and starts at out[s_gbase[p]].  Ends with a barrier.
// Every store that can be is a 16-byte store to a 16-byte aligned DESTINATION: the vector slot anchored at stage index k0
// is shifted back by the run's misalignment s = dest(k0) % V, so it reads V (unaligned) elements from shared memory and
// writes one aligned vector.  Only the elements whose aligned destination vector crosses the run's ends (< 2V per run)
// leave one by one.  (The first version stored aligned STAGE vectors and fell back to per-element loops for whole
// misaligned runs: the profiler counted about twice the ideal store sectors and DRAM writes.)
// `out_of(p)` is the array partition p's run goes to: one array for every partition (ps_store), or one per partition
// (hash.cu's split into owned tables); each must be 16-byte aligned.
template <typename T, int TILE, typename OutOf>
__device__ __forceinline__ void ps_store_to(const OutOf& out_of, const T* stage, int tile_n, const uint8_t* s_owner, const int32_t* s_start,
                                            const int32_t* s_gbase) {
  constexpr int V = sizeof(T) >= 16 ? 1 : 16 / (int)sizeof(T);
  // fixed trip count, fully unrolled: the iterations are independent and their shared-memory loads and global stores overlap.
  // (With the runtime bound `k0 < tile_n` the compiler unrolled this loop in one build and not in the next, and the kernel's
  // speed changed with an unrelated header change.)
  constexpr int ITERS = TILE / (PT_NT * V);
#pragma unroll
  for (int it = 0; it < ITERS; it++) {
    const int k0 = (it * PT_NT + (int)threadIdx.x) * V;
    if (k0 >= tile_n) continue;
    if (V == 1) { const int p = s_owner[k0]; __stcs(&out_of(p)[(int64_t)s_gbase[p] + (k0 - s_start[p])], stage[k0]); continue; }
    {
      const int p = s_owner[k0];
      const int64_t c = (int64_t)s_gbase[p] - s_start[p];       // dest(k) = k + c inside run p
      const int kk = k0 - (int)((k0 + c) % V);
      if (kk >= s_start[p] && kk + V <= s_start[p + 1]) {
        // whole sectors, never touched again: streaming store.  The boundary elements below keep the default policy: their
        // sector is completed by the neighbouring tile's run, and the kernel's DRAM writes depend on those half-written
        // sectors still being in L2 when the other half arrives
        __stcs(reinterpret_cast<uint4*>(out_of(p) + (kk + c)), pack16<T>(stage + kk));
      }
    }
#pragma unroll
    for (int i = 0; i < V; i++) {
      const int e = k0 + i;
      if (e >= tile_n) break;
      const int q = s_owner[e];
      const int64_t c = (int64_t)s_gbase[q] - s_start[q];
      const int kk = e - (int)((e + c) % V);
      if (!(kk >= s_start[q] && kk + V <= s_start[q + 1])) out_of(q)[e + c] = stage[e];
    }
  }
  __syncthreads();
}
template <typename T>
struct SameOut {
  T* __restrict__ p;
  __device__ __forceinline__ T* operator()(int) const { return p; }
};
template <typename T, int TILE>
__device__ __forceinline__ void ps_store(T* __restrict__ out, const T* stage, int tile_n, const uint8_t* s_owner, const int32_t* s_start,
                                         const int32_t* s_gbase) {
  ps_store_to<T, TILE>(SameOut<T>{out}, stage, tile_n, s_owner, s_start, s_gbase);
}
#endif

}  // namespace b2
