// hash.cu — a9: Spark-compatible Murmur3 (Hash.murmurHash32), pmod partition ids and Table.partition.
// Reference: GpuMurmur3Hash.compute (HashFunctions.scala:196-209), GpuHashPartitioner
// .hashPartitionAndClose (GpuHashPartitioningBase.scala:36-54, seed 42 at :100),
// GpuPartitioning.sliceInternalOnGpuAndClose (GpuPartitioning.scala:66-99), HashUtils.normalizeInput
// (shims/HashUtils.scala:53-77: -0.0 -> 0.0 before hashing).  The algorithm itself is Spark's
// org.apache.spark.unsafe.hash.Murmur3_x86_32 + HashExpression per-type rules (external spec;
// restated in oracle/spark_hash.py and pinned there by known answers).
//
// One kernel hashes all key columns (chained: the hash of column i seeds column i+1; a NULL leaves
// the running hash unchanged), applies pmod and writes the partition id; Table.partition is then a
// stable one- or two-digit radix split (sort.cu) followed by the fused multi-column gather.
#include "partition.cuh"
#include "prim.cuh"
#include "rowops.cuh"
#include "murmur.cuh"
#include <algorithm>

namespace b2 {

// out[i] = murmur3(keys of row i, seed); when nparts > 0, out[i] = pmod(hash, nparts)
__global__ void murmur_kernel(const __grid_constant__ KeyCols keys, int64_t n, uint32_t seed, int32_t nparts, int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t h = seed;
    for (int c = 0; c < keys.n; c++) h = murmur_col(keys.c[c], i, h);
    int32_t v = (int32_t)h;
    if (nparts > 0) { v = v % nparts; if (v < 0) v += nparts; }
    out[i] = v;
  }
}

__global__ void pid_keys_kernel(const int32_t* __restrict__ pids, int64_t n, uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = (uint64_t)(uint32_t)pids[i];
    vals[i] = (int32_t)i;
  }
}
__global__ void part_hist_kernel(const int32_t* __restrict__ pids, int64_t n, int32_t nparts, int32_t* __restrict__ counts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t p = pids[i];
    if (p >= 0 && p < nparts) atomicAdd(&counts[p], 1);
  }
}

int radix_sort_pairs(uint64_t* keys_a, int32_t* vals_a, uint64_t* keys_b, int32_t* vals_b, int64_t n, int nbytes);
Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols);

// ---- direct stable partition (<= 1024 partitions) -------------------------------------------------------------
// Two passes over the partition ids and ONE over the payload: per-tile histogram -> exclusive scan of the
// partition-major [partition][tile] counts -> every tile recomputes stable ranks (warp match_any + per-warp counts in
// shared memory, 256 rows at a time in row order) and writes each fixed-width NOT NULL column straight to its final
// place.  Reads are coalesced, writes are coalesced per run of equal ids.  Other columns (strings, nullable) go
// through the gather map the same kernel can emit.  Replaces id->key expansion + radix pass + random-read gather.
// PT_NT, PT_TILE, part_tile_hist_kernel, ps_store: partition.cuh
// Where a row's partition id comes from: an id array (Table.partition), or a digit of a 32-bit hash array (the radix group-by's
// passes, which move that hash array anyway: no separate digit pass and no id array)
struct PidArray {
  const int32_t* p;
  __device__ __forceinline__ int32_t operator()(int64_t i) const { return p[i]; }
};
struct HashDigit {
  const uint32_t* h;
  int shift;
  uint32_t mask;
  // default cache policy: the scatter moves the hash array itself right after, and that read should hit L2
  __device__ __forceinline__ int32_t operator()(int64_t i) const { return (int32_t)((h[i] >> shift) & mask); }
};

__global__ void __launch_bounds__(PT_NT) part_scatter_kernel(const int32_t* __restrict__ pids, int64_t n, int32_t nparts, int64_t ntiles,
                                                             const int32_t* __restrict__ base, const __grid_constant__ ScatterCols sc,
                                                             int32_t* __restrict__ map_out) {
  __shared__ int32_t run[PT_MAXP];              // next free output row of partition p for this tile
  __shared__ uint16_t wcnt[PT_NT / 32][PT_MAXP];  // rows of partition p per warp in the current 256-row step
  const int64_t tile = blockIdx.x;
  for (int p = threadIdx.x; p < nparts; p += PT_NT) {
    run[p] = base[(int64_t)p * ntiles + tile];
    for (int w = 0; w < PT_NT / 32; w++) wcnt[w][p] = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int j = 0; j < PT_STEPS; j++) {
    const int64_t i = tile * PT_TILE + (int64_t)j * PT_NT + threadIdx.x;
    int32_t p = -1;
    if (i < n) { p = pids[i]; if ((uint32_t)p >= (uint32_t)nparts) p = -1; }
    const uint32_t mask = __match_any_sync(0xffffffffu, p);
    const int rank = __popc(mask & ((1u << lane) - 1u));
    const int cnt = __popc(mask);
    if (p >= 0 && rank == 0) wcnt[w][p] = (uint16_t)cnt;
    __syncthreads();
    int32_t dest = 0;
    if (p >= 0) {
      int pre = 0;
      for (int w2 = 0; w2 < w; w2++) pre += wcnt[w2][p];
      dest = run[p] + pre + rank;
    }
    __syncthreads();
    if (p >= 0 && rank == 0) { atomicAdd(&run[p], cnt); wcnt[w][p] = 0; }
    if (p >= 0) {
      for (int c = 0; c < sc.n; c++) {
        switch (sc.width[c]) {
          case 1: reinterpret_cast<uint8_t*>(sc.out[c])[dest] = reinterpret_cast<const uint8_t*>(sc.in[c])[i]; break;
          case 2: reinterpret_cast<uint16_t*>(sc.out[c])[dest] = reinterpret_cast<const uint16_t*>(sc.in[c])[i]; break;
          case 4: reinterpret_cast<uint32_t*>(sc.out[c])[dest] = reinterpret_cast<const uint32_t*>(sc.in[c])[i]; break;
          case 8: reinterpret_cast<uint64_t*>(sc.out[c])[dest] = reinterpret_cast<const uint64_t*>(sc.in[c])[i]; break;
          default: reinterpret_cast<uint4*>(sc.out[c])[dest] = reinterpret_cast<const uint4*>(sc.in[c])[i]; break;
        }
      }
      if (map_out) map_out[dest] = (int32_t)i;
    }
    __syncthreads();
  }
}


// Stable multi-array scatter for <= 256 partitions, the workhorse of the radix group-by passes.  Ranks are computed like the
// radix sort's scatter (sort.cu): each warp owns 512 consecutive rows and ranks them 32 at a time with match_any against
// per-warp running counts (no block barrier inside the loop), one cross-warp scan gives every row its position in the
// tile's partition-sorted order.  Each array is then staged through shared memory in that order, so a partition's run
// leaves the SM as consecutive addresses (full sectors) instead of one scattered 8-byte store per row.
constexpr int PS_WARP_ITEMS = PT_TILE / PS_WARPS;
template <typename T>
__device__ __forceinline__ void ps_move(const T* __restrict__ in, T* __restrict__ out, T* stage, const uint16_t* lpos, int64_t wbase, int64_t n, int tile_n,
                                        const uint8_t* s_owner, const int32_t* s_start, const int32_t* s_gbase) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    if (i < n) stage[lpos[r]] = __ldcs(&in[i]);   // read once: evict-first, so the stream does not push the partially written sectors out of L2
  }
  __syncthreads();
  ps_store<T, PT_TILE>(out, stage, tile_n, s_owner, s_start, s_gbase);
}
__global__ void __launch_bounds__(PT_NT, 4) part_scatter2_kernel(const HashDigit pids, int64_t n, int32_t nparts, int64_t ntiles,
                                                              const int32_t* __restrict__ base, const __grid_constant__ ScatterCols sc) {
  extern __shared__ __align__(16) char ps_stage[];    // PT_TILE x widest array
  __shared__ uint32_t s_wh[PS_WARPS][256];
  __shared__ int32_t s_start[257], s_gbase[256];
  __shared__ uint8_t s_owner[PT_TILE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tile = blockIdx.x;
  const int tile_n = (int)min((int64_t)PT_TILE, n - tile * PT_TILE);
  for (int k = threadIdx.x; k < PS_WARPS * 256; k += PT_NT) (&s_wh[0][0])[k] = 0;
  __syncthreads();
  const int64_t wbase = tile * PT_TILE + (int64_t)warp * PS_WARP_ITEMS;
  uint8_t pid[PT_STEPS];
  uint16_t lpos[PT_STEPS];
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    const bool in = i < n;
    const uint32_t d = in ? (uint32_t)pids(i) : 256u + lane;   // out-of-range lanes match nobody
    const uint32_t m = __match_any_sync(0xffffffffu, d);
    const uint32_t before = __popc(m & ((1u << lane) - 1u));
    uint32_t prev = 0;
    if (in) prev = s_wh[warp][d];
    __syncwarp();
    if (in && before == 0) s_wh[warp][d] = prev + __popc(m);
    __syncwarp();
    pid[r] = (uint8_t)d;
    lpos[r] = (uint16_t)(prev + before);
  }
  __syncthreads();
  {  // partition d = threadIdx.x: exclusive offsets of the warps inside the partition's run, run length, global base
    const int d = threadIdx.x;
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < PS_WARPS; w++) { const uint32_t c = s_wh[w][d]; s_wh[w][d] = run; run += c; }
    s_start[d + 1] = (int32_t)run;     // counts for now
    s_gbase[d] = d < nparts ? base[(int64_t)d * ntiles + tile] : 0;
  }
  __syncthreads();
  if (threadIdx.x < 32) {   // exclusive scan of the 256 run lengths (8 per lane)
    int32_t c[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { c[k] = s_start[lane * 8 + k + 1]; sum += c[k]; }
    int32_t inc = sum;
    for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    int32_t runx = inc - sum;
#pragma unroll
    for (int k = 0; k < 8; k++) { s_start[lane * 8 + k] = runx; runx += c[k]; }
    if (lane == 31) s_start[256] = runx;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    if (i < n) {
      const int p = pid[r];
      lpos[r] = (uint16_t)(s_start[p] + s_wh[warp][p] + lpos[r]);
      s_owner[lpos[r]] = (uint8_t)p;
    }
  }
  __syncthreads();
  for (int c = 0; c < sc.n; c++) {
    switch (sc.width[c]) {
      case 1: ps_move<uint8_t>((const uint8_t*)sc.in[c], (uint8_t*)sc.out[c], (uint8_t*)ps_stage, lpos, wbase, n, tile_n, s_owner, s_start, s_gbase); break;
      case 2: ps_move<uint16_t>((const uint16_t*)sc.in[c], (uint16_t*)sc.out[c], (uint16_t*)ps_stage, lpos, wbase, n, tile_n, s_owner, s_start, s_gbase); break;
      case 4: ps_move<uint32_t>((const uint32_t*)sc.in[c], (uint32_t*)sc.out[c], (uint32_t*)ps_stage, lpos, wbase, n, tile_n, s_owner, s_start, s_gbase); break;
      case 8: ps_move<uint64_t>((const uint64_t*)sc.in[c], (uint64_t*)sc.out[c], (uint64_t*)ps_stage, lpos, wbase, n, tile_n, s_owner, s_start, s_gbase); break;
      default: ps_move<uint4>((const uint4*)sc.in[c], (uint4*)sc.out[c], (uint4*)ps_stage, lpos, wbase, n, tile_n, s_owner, s_start, s_gbase); break;
    }
  }
}

static Table* partition_table_direct(const Table* t, const int32_t* d_pids, int32_t nparts, int32_t* offsets_out) {
  const int64_t n = t->rows;
  const int64_t ntiles = (n + PT_TILE - 1) / PT_TILE;
  const int64_t cells = (int64_t)nparts * ntiles;
  DevBuf cnt((size_t)(cells + 1) * 4);
  launch("part_tile_hist_kernel", part_tile_hist_kernel<PidArray>, (int)ntiles, PT_NT, 0, stream(), PidArray{d_pids}, n, nparts, ntiles, cnt.as<int32_t>());
  DevBuf sums = exclusive_scan<int32_t, int32_t>(cnt.as<int32_t>(), cnt.as<int32_t>(), cells, true);
  std::vector<int32_t> h(nparts + 1, 0);
  CUDA_CHECK(cudaMemcpy2DAsync(h.data(), 4, cnt.p, (size_t)ntiles * 4, 4, (size_t)nparts, cudaMemcpyDeviceToHost, stream()));
  d2h(&h[nparts], cnt.as<int32_t>() + cells, 1);
  // outputs: fixed-width NOT NULL columns are written by the scatter kernel itself, the rest through the gather map
  ColsGuard outs;
  outs.v.resize(t->cols.size(), nullptr);
  ScatterCols sc; memset(&sc, 0, sizeof(sc));
  std::vector<int> via_map;
  for (size_t c = 0; c < t->cols.size(); c++) {
    const Column* ic = t->cols[c];
    if (ic->dtype != B2_STRING && !ic->nullable() && sc.n < PT_MAXC) {
      Column* oc = new_column(ic->dtype, ic->scale, n, false);
      outs.v[c] = oc;
      sc.width[sc.n] = dtype_width(ic->dtype); sc.in[sc.n] = ic->data.p; sc.out[sc.n] = oc->data.p; sc.n++;
    } else via_map.push_back((int)c);
  }
  DevBuf map;
  if (!via_map.empty()) map = DevBuf((size_t)n * 4);
  launch("part_scatter_kernel", part_scatter_kernel, (int)ntiles, PT_NT, 0, stream(), d_pids, n, nparts, ntiles, cnt.as<int32_t>(), sc, map.as<int32_t>());
  sync();
  if (h[nparts] != n) throw Error(B2_ERR_INVALID, "partition ids out of range");
  for (int p = 0; p <= nparts; p++) offsets_out[p] = h[p];
  if (!via_map.empty()) {
    Table* g = gather_table(t, map.as<int32_t>(), n, false, &via_map);
    for (size_t k = 0; k < via_map.size(); k++) { outs.v[via_map[k]] = g->cols[k]; col_incref(g->cols[k]); }
    table_release(g);
  }
  return new_table(outs.release());
}

// raw-array form (radix group-by, agg.cu): stable scatter of up to PT_MAXC fixed-width arrays by the digit
// (d_hash[i] >> shift) & (2^bits - 1), bits <= 8
void partition_scatter_by_hash(const uint32_t* d_hash, int shift, int bits, int64_t n, const ScatterCols& sc) {
  if (n == 0) return;
  B2_CHECK(bits >= 1 && bits <= 8, "partition_scatter_by_hash: 1..8 digit bits");
  const int32_t nparts = 1 << bits;
  const HashDigit pid{d_hash, shift, (uint32_t)nparts - 1u};
  const int64_t ntiles = (n + PT_TILE - 1) / PT_TILE;
  const int64_t cells = (int64_t)nparts * ntiles;
  DevBuf cnt((size_t)(cells + 1) * 4);
  launch("part_tile_hist_kernel", part_tile_hist_kernel<HashDigit>, (int)ntiles, PT_NT, 0, stream(), pid, n, nparts, ntiles, cnt.as<int32_t>());
  DevBuf sums = exclusive_scan<int32_t, int32_t>(cnt.as<int32_t>(), cnt.as<int32_t>(), cells, true);
  int maxw = 1;
  for (int c = 0; c < sc.n; c++) maxw = std::max(maxw, sc.width[c]);
  launch("part_scatter2_kernel", part_scatter2_kernel, (int)ntiles, PT_NT, PT_TILE * maxw, stream(), pid, n, nparts, ntiles, cnt.as<int32_t>(), sc);
  sync();   // cnt / sums are freed on return
}

// ---- split into owned tables (GpuBatchSubPartitioner: hashPartition + contiguousSplit in one pass) -------------------------
// Count pass: bucket[i] = pmod(murmur3(keys of row sel ? sel[i] : i, seed), nparts) (one byte) and the per-(bucket, tile) counts.
// After the exclusive scan of those counts, base[p * ntiles + tile] is where the tile's run of bucket p starts in the bucket-major
// order of all rows, and base[p * ntiles] where bucket p starts.
__global__ void __launch_bounds__(PT_NT) hash_split_count_kernel(const __grid_constant__ KeyCols keys, const int32_t* __restrict__ sel, int64_t n,
                                                                 uint32_t seed, int32_t nparts, int64_t ntiles, uint8_t* __restrict__ bucket,
                                                                 int32_t* __restrict__ tile_cnt) {
  __shared__ int32_t h[256];
  for (int p = threadIdx.x; p < nparts; p += PT_NT) h[p] = 0;
  __syncthreads();
  const int64_t tile = blockIdx.x;
  for (int j = 0; j < PT_STEPS; j++) {
    const int64_t i = tile * PT_TILE + (int64_t)j * PT_NT + threadIdx.x;
    if (i < n) {
      const int64_t r = sel ? (int64_t)sel[i] : i;
      uint32_t hv = seed;
      for (int c = 0; c < keys.n; c++) hv = murmur_col(keys.c[c], r, hv);
      int32_t p = (int32_t)hv % nparts;
      if (p < 0) p += nparts;
      bucket[i] = (uint8_t)p;
      atomicAdd(&h[p], 1);
    }
  }
  __syncthreads();
  for (int p = threadIdx.x; p < nparts; p += PT_NT) tile_cnt[(int64_t)p * ntiles + tile] = h[p];
}

struct SplitCol { const void* in; const uint32_t* in_valid; int32_t width; int32_t pad; };

template <typename T>
struct BucketOut {
  void* const* o;
  __device__ __forceinline__ T* operator()(int p) const { return reinterpret_cast<T*>(o[p]); }
};
template <typename T>
__device__ __forceinline__ void hs_move(const T* __restrict__ in, const int32_t* __restrict__ sel, void* const* s_out, T* stage, const uint16_t* s_lpos,
                                        int64_t tbase, int tile_n, const uint8_t* s_owner, const int32_t* s_start, const int32_t* s_gbase) {
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int k = r * PT_NT + threadIdx.x;
    if (k < tile_n) stage[s_lpos[k]] = __ldcs(&in[sel ? (int64_t)sel[tbase + k] : tbase + k]);
  }
  __syncthreads();
  ps_store_to<T, PT_TILE>(BucketOut<T>{s_out}, stage, tile_n, s_owner, s_start, s_gbase);
}

// Scatter pass: ranks every row of the tile stably by its bucket byte (as part_scatter2_kernel does), then moves each fixed-width
// column through shared memory in bucket order and stores every run into its bucket's own array with aligned 16-byte vectors.
// Validity bits follow the same order: a bucket mask word that lies inside one run is stored, a word the run shares with a
// neighbouring tile's run is OR-ed into the zeroed mask.  map_out (strings present): the row id of every output row, bucket-major.
__global__ void __launch_bounds__(PT_NT, 2) hash_split_scatter_kernel(const uint8_t* __restrict__ bucket, const int32_t* __restrict__ sel, int64_t n,
                                                                   int32_t nparts, int64_t ntiles, const int32_t* __restrict__ base, int32_t ncols,
                                                                   const SplitCol* __restrict__ cols, void* const* __restrict__ outs,
                                                                   uint32_t* const* __restrict__ out_valid, int32_t* __restrict__ map_out) {
  extern __shared__ __align__(16) char ps_stage[];    // PT_TILE x widest column; the validity bits reuse it
  __shared__ uint32_t s_wh[PS_WARPS][256];
  __shared__ int32_t s_start[257], s_gbase[256], s_goff[256];
  __shared__ uint8_t s_owner[PT_TILE];
  __shared__ uint16_t s_lpos[PT_TILE];   // where row k of the tile sits in bucket order
  __shared__ void* s_out[256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t tile = blockIdx.x;
  const int tile_n = (int)min((int64_t)PT_TILE, n - tile * PT_TILE);
  for (int k = threadIdx.x; k < PS_WARPS * 256; k += PT_NT) (&s_wh[0][0])[k] = 0;
  __syncthreads();
  const int64_t tbase = tile * PT_TILE, wbase = tbase + (int64_t)warp * PS_WARP_ITEMS;
  uint8_t pid[PT_STEPS];
  uint16_t lpos[PT_STEPS];
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    const bool in = i < n;
    const uint32_t d = in ? (uint32_t)bucket[i] : 256u + lane;   // out-of-range lanes match nobody
    const uint32_t m = __match_any_sync(0xffffffffu, d);
    const uint32_t before = __popc(m & ((1u << lane) - 1u));
    uint32_t prev = 0;
    if (in) prev = s_wh[warp][d];
    __syncwarp();
    if (in && before == 0) s_wh[warp][d] = prev + __popc(m);
    __syncwarp();
    pid[r] = (uint8_t)d;
    lpos[r] = (uint16_t)(prev + before);
  }
  __syncthreads();
  {  // bucket d = threadIdx.x: offsets of the warps inside the bucket's run, run length, where the run starts in the bucket
    const int d = threadIdx.x;
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < PS_WARPS; w++) { const uint32_t c = s_wh[w][d]; s_wh[w][d] = run; run += c; }
    s_start[d + 1] = (int32_t)run;
    s_goff[d] = d < nparts ? base[(int64_t)d * ntiles + tile] : 0;
    s_gbase[d] = d < nparts ? s_goff[d] - base[(int64_t)d * ntiles] : 0;
  }
  __syncthreads();
  if (threadIdx.x < 32) {   // exclusive scan of the 256 run lengths (8 per lane)
    int32_t c[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { c[k] = s_start[lane * 8 + k + 1]; sum += c[k]; }
    int32_t inc = sum;
    for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    int32_t runx = inc - sum;
#pragma unroll
    for (int k = 0; k < 8; k++) { s_start[lane * 8 + k] = runx; runx += c[k]; }
    if (lane == 31) s_start[256] = runx;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < PT_STEPS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    if (i < n) {
      const int p = pid[r];
      const int pos = s_start[p] + (int)s_wh[warp][p] + lpos[r];
      s_lpos[i - tbase] = (uint16_t)pos;
      s_owner[pos] = (uint8_t)p;
      if (map_out) map_out[s_goff[p] + (pos - s_start[p])] = sel ? sel[i] : (int32_t)i;
    }
  }
  __syncthreads();
  for (int c = 0; c < ncols; c++) {
    const SplitCol col = cols[c];
    for (int p = threadIdx.x; p < nparts; p += PT_NT) s_out[p] = outs[(int64_t)c * nparts + p];
    __syncthreads();
    switch (col.width) {
      case 1: hs_move<uint8_t>((const uint8_t*)col.in, sel, s_out, (uint8_t*)ps_stage, s_lpos, tbase, tile_n, s_owner, s_start, s_gbase); break;
      case 2: hs_move<uint16_t>((const uint16_t*)col.in, sel, s_out, (uint16_t*)ps_stage, s_lpos, tbase, tile_n, s_owner, s_start, s_gbase); break;
      case 4: hs_move<uint32_t>((const uint32_t*)col.in, sel, s_out, (uint32_t*)ps_stage, s_lpos, tbase, tile_n, s_owner, s_start, s_gbase); break;
      case 8: hs_move<uint64_t>((const uint64_t*)col.in, sel, s_out, (uint64_t*)ps_stage, s_lpos, tbase, tile_n, s_owner, s_start, s_gbase); break;
      default: hs_move<uint4>((const uint4*)col.in, sel, s_out, (uint4*)ps_stage, s_lpos, tbase, tile_n, s_owner, s_start, s_gbase); break;
    }
    if (col.in_valid) {   // ends with a barrier like the moves, so s_out and the stage are free again afterwards
      uint8_t* s_bit = reinterpret_cast<uint8_t*>(ps_stage);
      for (int p = threadIdx.x; p < nparts; p += PT_NT) s_out[p] = out_valid[(int64_t)c * nparts + p];
#pragma unroll
      for (int r = 0; r < PT_STEPS; r++) {
        const int k = r * PT_NT + threadIdx.x;
        if (k < tile_n) s_bit[s_lpos[k]] = (uint8_t)bit_get(col.in_valid, sel ? (int64_t)sel[tbase + k] : tbase + k);
      }
      __syncthreads();
      for (int p = warp; p < nparts; p += PS_WARPS) {   // one warp per run; lane l builds bit l of each word with a ballot
        const int len = s_start[p + 1] - s_start[p];
        if (len == 0) continue;
        const int64_t g = s_gbase[p];
        uint32_t* ov = reinterpret_cast<uint32_t*>(s_out[p]);
        for (int64_t w = g >> 5; w <= (g + len - 1) >> 5; w++) {
          const int64_t b = w * 32 + lane;
          const bool v = b >= g && b < g + len && s_bit[s_start[p] + (int)(b - g)];
          const uint32_t word = __ballot_sync(0xffffffffu, v);
          if (lane == 0) {
            if (w * 32 >= g && w * 32 + 32 <= g + len) ov[w] = word;
            else if (word) atomicOr(&ov[w], word);
          }
        }
      }
      __syncthreads();
    }
  }
}

// rows of t (or the n rows sel names) -> nparts owned tables of the columns `keep`; nullptr for an empty part
std::vector<Table*> hash_split_table(const Table* t, const int32_t* d_sel, int64_t n, const int32_t* key_cols, int nkeys, uint32_t seed,
                                     int nparts, const std::vector<int>& keep) {
  B2_CHECK(nparts >= 2 && nparts <= 256, "hash split: 2 to 256 parts");
  B2_CHECK(nkeys >= 1 && !keep.empty(), "hash split: at least one key and one kept column");
  const KeyCols keys = key_cols_of(t, key_cols, nkeys);
  for (int c : keep) B2_CHECK(c >= 0 && c < (int)t->cols.size(), "hash split: kept column out of range");
  if (n > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "hash split of more than 2^31-1 rows");
  std::vector<Table*> out(nparts, nullptr);
  if (n == 0) return out;
  const int64_t ntiles = (n + PT_TILE - 1) / PT_TILE;
  const int64_t cells = (int64_t)nparts * ntiles;
  DevBuf bucket((size_t)n), cnt((size_t)(cells + 1) * 4);
  launch("hash_split_count_kernel", hash_split_count_kernel, (int)ntiles, PT_NT, 0, stream(), keys, d_sel, n, seed, nparts, ntiles,
         bucket.as<uint8_t>(), cnt.as<int32_t>());
  DevBuf sums = exclusive_scan<int32_t, int32_t>(cnt.as<int32_t>(), cnt.as<int32_t>(), cells, true);
  std::vector<int32_t> start(nparts + 1, 0);
  CUDA_CHECK(cudaMemcpy2DAsync(start.data(), 4, cnt.p, (size_t)ntiles * 4, 4, (size_t)nparts, cudaMemcpyDeviceToHost, stream()));
  d2h(&start[nparts], cnt.as<int32_t>() + cells, 1);
  sync();
  const int nk = (int)keep.size();
  ColsGuard all;   // [p * nk + k]
  all.v.resize((size_t)nparts * nk, nullptr);
  std::vector<SplitCol> fixed;
  std::vector<void*> outs, outv;
  std::vector<int> via_map;   // output positions of the STRING columns
  int maxw = 1;
  for (int k = 0; k < nk; k++) {
    const Column* ic = t->cols[keep[k]];
    if (ic->dtype == B2_STRING) { via_map.push_back(k); continue; }
    fixed.push_back(SplitCol{ic->data.p, ic->validity(), dtype_width(ic->dtype), 0});
    maxw = std::max(maxw, dtype_width(ic->dtype));
    for (int p = 0; p < nparts; p++) {
      const int64_t rows = start[p + 1] - start[p];
      Column* oc = nullptr;
      if (rows) {
        oc = new_column(ic->dtype, ic->scale, rows, ic->nullable());
        all.v[(size_t)p * nk + k] = oc;
        if (oc->valid.p) CUDA_CHECK(cudaMemsetAsync(oc->valid.p, 0, oc->valid.bytes, stream()));
      }
      outs.push_back(oc ? oc->data.p : nullptr);
      outv.push_back(oc ? oc->valid.p : nullptr);
    }
  }
  DevBuf map;
  if (!via_map.empty()) map = DevBuf((size_t)n * 4);
  if (!fixed.empty() || map.p) {
    const size_t fb = fixed.size() * sizeof(SplitCol), pb = outs.size() * sizeof(void*);
    DevBuf desc(std::max<size_t>(fb + 2 * pb, 1));
    if (fb) {
      h2d_bytes(desc.p, fixed.data(), fb);
      h2d_bytes((char*)desc.p + fb, outs.data(), pb);
      h2d_bytes((char*)desc.p + fb + pb, outv.data(), pb);
    }
    launch("hash_split_scatter_kernel", hash_split_scatter_kernel, (int)ntiles, PT_NT, (size_t)PT_TILE * maxw, stream(), bucket.as<uint8_t>(), d_sel, n,
           nparts, ntiles, cnt.as<int32_t>(), (int32_t)fixed.size(), (const SplitCol*)desc.p, (void* const*)((char*)desc.p + fb),
           (uint32_t* const*)((char*)desc.p + fb + pb), map.as<int32_t>());
  }
  if (!via_map.empty()) {
    std::vector<int> str_cols;
    for (int k : via_map) str_cols.push_back(keep[k]);
    for (int p = 0; p < nparts; p++) {
      const int64_t rows = start[p + 1] - start[p];
      if (!rows) continue;
      Table* g = gather_table(t, map.as<int32_t>() + start[p], rows, false, &str_cols);
      for (size_t q = 0; q < via_map.size(); q++) { all.v[(size_t)p * nk + via_map[q]] = g->cols[q]; col_incref(g->cols[q]); }
      table_release(g);
    }
  }
  for (int p = 0; p < nparts; p++) {
    if (start[p + 1] == start[p]) continue;
    std::vector<Column*> cs(all.v.begin() + (size_t)p * nk, all.v.begin() + (size_t)(p + 1) * nk);
    for (int k = 0; k < nk; k++) all.v[(size_t)p * nk + k] = nullptr;
    out[p] = new_table(std::move(cs));   // the columns have the part's length: cannot throw
  }
  return out;
}

// Table.partition: stable reorder so each partition is contiguous + partition start offsets
Table* partition_table(const Table* t, const int32_t* d_pids, int32_t nparts, int32_t* offsets_out) {
  const int64_t n = t->rows;
  B2_CHECK(nparts >= 1, "need at least one partition");
  if (nparts <= PT_MAXP && n >= PT_TILE) return partition_table_direct(t, d_pids, nparts, offsets_out);
  DevBuf counts((size_t)nparts * 4);
  CUDA_CHECK(cudaMemsetAsync(counts.p, 0, counts.bytes, stream()));
  std::vector<int32_t> h(nparts, 0);
  if (n) {
    launch(part_hist_kernel, grid_for(n, 256), 256, 0, stream(), d_pids, n, nparts, counts.as<int32_t>());
    d2h(h.data(), counts.p, nparts);
  }
  DevBuf ka((size_t)std::max<int64_t>(n, 1) * 8), kb((size_t)std::max<int64_t>(n, 1) * 8);
  DevBuf va((size_t)std::max<int64_t>(n, 1) * 4), vb((size_t)std::max<int64_t>(n, 1) * 4);
  int which = 0;
  if (n) {
    launch(pid_keys_kernel, grid_for(n, 256), 256, 0, stream(), d_pids, n, ka.as<uint64_t>(), va.as<int32_t>());
    int nbytes = nparts <= 256 ? 1 : (nparts <= 65536 ? 2 : 4);
    which = radix_sort_pairs(ka.as<uint64_t>(), va.as<int32_t>(), kb.as<uint64_t>(), vb.as<int32_t>(), n, nbytes);
  }
  sync();
  int64_t run = 0;
  for (int p = 0; p < nparts; p++) { offsets_out[p] = (int32_t)run; run += h[p]; }
  offsets_out[nparts] = (int32_t)run;
  if (run != n) throw Error(B2_ERR_INVALID, "partition ids out of range");
  return gather_table(t, which ? vb.as<int32_t>() : va.as<int32_t>(), n, false, nullptr);
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_murmur3(b2_handle table, const int32_t* cols, int32_t ncols, int32_t seed, b2_handle* out_int32_col) {
  B2_TRY
  Table* t = table_from(table);
  KeyCols keys = key_cols_of(t, cols, ncols);
  ColGuard out(new_column(B2_INT32, 0, t->rows, false));
  if (t->rows) launch(murmur_kernel, grid_for(t->rows, 256), 256, 0, stream(), keys, t->rows, (uint32_t)seed, 0, out.c->data.as<int32_t>());
  *out_int32_col = to_handle(out.release());
  B2_CATCH
}

int b2_hash_partition(b2_handle table, const int32_t* key_cols, int32_t nkeys, int32_t seed, int32_t num_partitions,
                      b2_handle* out_table, int32_t* offsets_out) {
  B2_TRY
  Table* t = table_from(table);
  B2_CHECK(num_partitions >= 1, "need at least one partition");
  KeyCols keys = key_cols_of(t, key_cols, nkeys);
  DevBuf pids((size_t)std::max<int64_t>(t->rows, 1) * 4);
  if (t->rows) launch("murmur_pmod_kernel", murmur_kernel, grid_for(t->rows, 256), 256, 0, stream(), keys, t->rows, (uint32_t)seed, num_partitions, pids.as<int32_t>());
  *out_table = to_handle(partition_table(t, pids.as<int32_t>(), num_partitions, offsets_out));
  B2_CATCH
}

int b2_hash_split(b2_handle table, b2_handle sel, const int32_t* key_cols, int32_t nkeys, int32_t seed, int32_t num_parts,
                  const int32_t* keep_cols, int32_t nkeep, b2_handle* out_tables) {
  B2_TRY
  Table* t = table_from(table);
  const Column* s = sel ? col_from(sel) : nullptr;
  B2_CHECK(!s || (s->dtype == B2_INT32 && !s->nullable()), "selection vector must be INT32 without NULLs");
  std::vector<int> keep;
  if (keep_cols) keep.assign(keep_cols, keep_cols + nkeep);
  else for (int c = 0; c < (int)t->cols.size(); c++) keep.push_back(c);
  std::vector<Table*> parts = hash_split_table(t, s ? s->data.as<int32_t>() : nullptr, s ? s->size : t->rows, key_cols, nkeys, (uint32_t)seed,
                                               num_parts, keep);
  for (int p = 0; p < num_parts; p++) out_tables[p] = to_handle(parts[p]);
  B2_CATCH
}

int b2_partition_by_ids(b2_handle table, b2_handle int32_part_ids, int32_t num_partitions, b2_handle* out_table, int32_t* offsets_out) {
  B2_TRY
  Table* t = table_from(table);
  Column* p = col_from(int32_part_ids);
  B2_CHECK(p->dtype == B2_INT32 && p->size == t->rows, "partition ids must be INT32, one per row");
  *out_table = to_handle(partition_table(t, p->data.as<int32_t>(), num_partitions, offsets_out));
  B2_CATCH
}

}  // extern "C"
