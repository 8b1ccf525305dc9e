// prim.cuh — hand-written device-wide primitives shared by the operators (no CUB/Thrust):
// exclusive prefix sum (reduce-then-scan, 3 launches), used for string gathers, partition
// offsets and radix-sort digit offsets.
#pragma once
#include "common.cuh"

namespace b2 {

// stable multi-array partition scatter (hash.cu): up to PT_MAXC fixed-width arrays moved by one kernel
constexpr int PT_MAXC = 8;
struct ScatterCols {
  int32_t n;
  int32_t width[PT_MAXC];
  const void* in[PT_MAXC];
  void* out[PT_MAXC];
};
// the partition of row i is the digit (d_hash[i] >> shift) & (2^bits - 1), bits <= 8
void partition_scatter_by_hash(const uint32_t* d_hash, int shift, int bits, int64_t n, const ScatterCols& sc);

#ifdef __CUDACC__
constexpr int SCAN_NT = 256;
constexpr int SCAN_ITEMS = 8;                      // items per thread
constexpr int SCAN_TILE = SCAN_NT * SCAN_ITEMS;   // 2048 items per CTA

template <typename TIn>
__global__ void __launch_bounds__(SCAN_NT) scan_reduce_kernel(const TIn* __restrict__ in, int64_t n, int64_t* __restrict__ tile_sums) {
  __shared__ int64_t s_w[SCAN_NT / 32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
  int64_t acc = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    int64_t i = base + k * SCAN_NT + threadIdx.x;
    if (i < n) acc += (int64_t)in[i];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int w = 0; w < SCAN_NT / 32; w++) t += s_w[w];
    tile_sums[blockIdx.x] = t;
  }
}

// single CTA: exclusive scan of up to a few hundred thousand tile sums, writes total at [ntiles]
static __global__ void __launch_bounds__(1024) scan_tiles_kernel(int64_t* __restrict__ tile_sums, int64_t ntiles) {
  __shared__ int64_t s_w[32];
  __shared__ int64_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < ntiles; base += 1024) {
    int64_t i = base + threadIdx.x;
    int64_t v = i < ntiles ? tile_sums[i] : 0;
    int64_t inc = v;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      int64_t w = s_w[lane], winc = w;
      for (int o = 1; o < 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
      s_w[lane] = winc - w;
    }
    __syncthreads();
    const int64_t carry = s_carry;
    if (i < ntiles) tile_sums[i] = carry + s_w[warp] + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + s_w[warp] + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) tile_sums[ntiles] = s_carry;
}

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(SCAN_NT) scan_final_kernel(const TIn* __restrict__ in, TOut* __restrict__ out, int64_t n,
                                                             const int64_t* __restrict__ tile_sums, bool write_total) {
  __shared__ int64_t s_w[SCAN_NT / 32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;  // blocked arrangement
  int64_t v[SCAN_ITEMS];
  int64_t sum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = (base + k < n) ? (int64_t)in[base + k] : 0; sum += v[k]; }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t inc = sum;
  for (int o = 1; o < 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  if (warp == 0 && lane < SCAN_NT / 32) {
    int64_t w = s_w[lane], winc = w;
    for (int o = 1; o < SCAN_NT / 32; o <<= 1) { int64_t t = __shfl_up_sync(0xffu, winc, o); if (lane >= o) winc += t; }
    s_w[lane] = winc - w;
  }
  __syncthreads();
  int64_t run = tile_sums[blockIdx.x] + s_w[warp] + inc - sum;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < n) out[base + k] = (TOut)run;
    run += v[k];
  }
  if (write_total && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = (TOut)tile_sums[gridDim.x];
}

// out[i] = sum(in[0..i)), optionally out[n] = total.  in and out may alias when types match in size.
// Returns a device pointer holder whose [ntiles] element is the grand total (int64).
template <typename TIn, typename TOut>
inline DevBuf exclusive_scan(const TIn* in, TOut* out, int64_t n, bool write_total) {
  int64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  if (ntiles < 1) ntiles = 1;
  DevBuf sums((size_t)(ntiles + 1) * 8);
  if (n == 0) {
    CUDA_CHECK(cudaMemsetAsync(sums.p, 0, sums.bytes, stream()));
    if (write_total) CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(TOut), stream()));
    return sums;
  }
  launch(scan_reduce_kernel<TIn>, (int)ntiles, SCAN_NT, 0, stream(), in, n, sums.as<int64_t>());
  launch(scan_tiles_kernel, 1, 1024, 0, stream(), sums.as<int64_t>(), ntiles);
  launch(scan_final_kernel<TIn, TOut>, (int)ntiles, SCAN_NT, 0, stream(), in, out, n, sums.as<int64_t>(), write_total);
  return sums;
}
#endif

}  // namespace b2
