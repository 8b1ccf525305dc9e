// sort.cu — a8: Table.sortOrder / orderBy / merge / upperBound / lowerBound and GpuTopN.
// Reference: SortUtils.scala:172-218, 249-342, 373-400 (GpuSorter), SortUtils.getOrder :38-43
// (asc(idx, nullsFirst) / desc(idx, nullsLast)), GpuSortExec.scala:87-165, limit.scala:234-330.
//
// The reference calls cudf's comparator-based multi-column sort and a separate gather.  Here the
// sort is an LSD radix sort over *normalised* keys: every key column is mapped to an
// order-preserving big-endian byte string (sign flip for integers/decimals, total-order transform
// for floats with -0.0 == 0.0 and NaN greatest, a leading null byte honouring nulls-first/last,
// descending = bitwise NOT, strings zero-padded + length), the row key is the concatenation, and
// 64-bit chunks of it are sorted from least to most significant with a stable 8-bit-digit radix
// pass (per-tile histograms -> scan -> ranked scatter; warp ranks via __match_any_sync).  Digits on
// which all rows agree are skipped.  Stable by construction (docs/compatibility.md:31-41 allows
// either, stableSort.enabled needs it).
#include <algorithm>
#include "prim.cuh"

namespace b2 {

constexpr int RS_NT = 256;
constexpr int RS_ITEMS = 16;
constexpr int RS_TILE = RS_NT * RS_ITEMS;  // 4096 items per CTA
constexpr int RS_WARPS = RS_NT / 32;
constexpr int RS_WARP_ITEMS = RS_TILE / RS_WARPS;  // 512 consecutive items per warp

// histogram of the first `ndigits` digits of the chunk in one read (shared-memory atomics; a
// match_any pre-aggregation was measured slower for 8-bit digits of random keys)
__global__ void __launch_bounds__(256) hist8_kernel(const uint64_t* __restrict__ keys, int64_t n, int ndigits, unsigned long long* __restrict__ hist) {
  __shared__ uint32_t s_h[8 * 256];
  for (int k = threadIdx.x; k < 8 * 256; k += blockDim.x) s_h[k] = 0;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t k = keys[i];
    for (int d = 0; d < ndigits; d++) atomicAdd(&s_h[d * 256 + ((k >> (8 * d)) & 255)], 1u);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ndigits * 256; k += blockDim.x)
    if (s_h[k]) atomicAdd(&hist[k], (unsigned long long)s_h[k]);
}

// per-tile histogram of one digit, stored digit-major: tile_hist[digit * ntiles + tile]
__global__ void __launch_bounds__(RS_NT) tile_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift,
                                                          int32_t* __restrict__ tile_hist, int64_t ntiles) {
  __shared__ uint32_t s_h[256];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * RS_TILE;
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    const int64_t i = base + k * RS_NT + threadIdx.x;
    if (i < n) atomicAdd(&s_h[(keys[i] >> shift) & 255], 1u);
  }
  __syncthreads();
  tile_hist[(int64_t)threadIdx.x * ntiles + blockIdx.x] = (int32_t)s_h[threadIdx.x];
}

// stable ranked scatter of (key, value) by one digit
__global__ void __launch_bounds__(RS_NT) scatter_kernel(const uint64_t* __restrict__ keys_in, const int32_t* __restrict__ vals_in,
                                                        uint64_t* __restrict__ keys_out, int32_t* __restrict__ vals_out, int64_t n,
                                                        int shift, const int64_t* __restrict__ tile_offsets, int64_t ntiles) {
  __shared__ uint32_t s_wh[RS_WARPS][256];  // per-warp digit counts, then exclusive offsets across warps
  __shared__ int64_t s_base[256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < RS_WARPS * 256; k += RS_NT) (&s_wh[0][0])[k] = 0;
  __syncthreads();
  const int64_t wbase = (int64_t)blockIdx.x * RS_TILE + (int64_t)warp * RS_WARP_ITEMS;
  uint64_t key[RS_ITEMS];
  uint16_t rank[RS_ITEMS];
#pragma unroll
  for (int r = 0; r < RS_ITEMS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    const bool in = i < n;
    key[r] = in ? keys_in[i] : 0;
    const uint32_t d = in ? (uint32_t)((key[r] >> shift) & 255) : 256u + lane;  // out-of-range lanes match nobody
    const uint32_t m = __match_any_sync(0xffffffffu, d);
    const uint32_t before = __popc(m & ((1u << lane) - 1u));
    uint32_t prev = 0;
    if (in) prev = s_wh[warp][d];
    __syncwarp();
    if (in && before == 0) s_wh[warp][d] = prev + __popc(m);  // one leader per distinct digit
    __syncwarp();
    rank[r] = (uint16_t)(prev + before);
  }
  __syncthreads();
  {  // exclusive scan across warps for digit = threadIdx.x, and fetch the tile's global base
    const int d = threadIdx.x;
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; w++) { uint32_t c = s_wh[w][d]; s_wh[w][d] = run; run += c; }
    s_base[d] = tile_offsets[(int64_t)d * ntiles + blockIdx.x];
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < RS_ITEMS; r++) {
    const int64_t i = wbase + r * 32 + lane;
    if (i < n) {
      const uint32_t d = (uint32_t)((key[r] >> shift) & 255);
      const int64_t o = s_base[d] + s_wh[warp][d] + rank[r];
      keys_out[o] = key[r];
      vals_out[o] = vals_in[i];
    }
  }
}

__global__ void iota32_kernel(int32_t* out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (int32_t)i;
}

// Sort (keys, vals) by bytes [0, nbytes) of keys (LSD, stable).  Buffers ping-pong; returns which
// pair holds the result (0 = a, 1 = b).
int radix_sort_pairs(uint64_t* keys_a, int32_t* vals_a, uint64_t* keys_b, int32_t* vals_b, int64_t n, int nbytes) {
  if (n <= 1) return 0;
  DevBuf hist(8 * 256 * 8);
  CUDA_CHECK(cudaMemsetAsync(hist.p, 0, hist.bytes, stream()));
  launch(hist8_kernel, grid_for(n, 256 * 8), 256, 0, stream(), keys_a, n, nbytes, hist.as<unsigned long long>());
  std::vector<unsigned long long> h(8 * 256);
  d2h(h.data(), hist.p, h.size());
  sync();
  const int64_t ntiles = (n + RS_TILE - 1) / RS_TILE;
  DevBuf th((size_t)256 * ntiles * 4), to((size_t)(256 * ntiles + 1) * 8);
  int cur = 0;
  for (int d = 0; d < nbytes; d++) {
    bool trivial = false;
    for (int b = 0; b < 256; b++)
      if (h[d * 256 + b] == (unsigned long long)n) trivial = true;
    if (trivial) continue;
    uint64_t* kin = cur ? keys_b : keys_a; int32_t* vin = cur ? vals_b : vals_a;
    uint64_t* kout = cur ? keys_a : keys_b; int32_t* vout = cur ? vals_a : vals_b;
    launch("radix_tile_hist_kernel", tile_hist_kernel, (int)ntiles, RS_NT, 0, stream(), kin, n, 8 * d, th.as<int32_t>(), ntiles);
    exclusive_scan<int32_t, int64_t>(th.as<int32_t>(), to.as<int64_t>(), 256 * ntiles, false);
    launch("radix_scatter_kernel", scatter_kernel, (int)ntiles, RS_NT, 0, stream(), kin, vin, kout, vout, n, 8 * d, to.as<int64_t>(), ntiles);
    cur ^= 1;
  }
  return cur;
}

// ------------------------------------------------------------------------------------------------
// key normalisation
constexpr int SORT_MAX_KEYS = 16;
struct SortCol {
  const void* data;
  const uint32_t* valid;
  const int32_t* offsets;
  int32_t dtype, width;
  int32_t ascending, nulls_first;
  int32_t key_off;    // first byte of this column inside the row key
  int32_t key_len;    // bytes (null byte included)
  int32_t has_null_byte;
  int32_t str_max;    // strings: padded length
};
struct SortPlan {
  int32_t ncols;
  int32_t key_bytes;
  SortCol c[SORT_MAX_KEYS];
};

// byte `b` (0 = most significant) of column c's normalised key for `row`
__device__ __forceinline__ uint32_t norm_byte(const SortCol& c, int64_t row, int b) {
  const bool valid = row_valid(c.valid, row);
  uint32_t out;
  if (c.has_null_byte && b == 0) {
    // nulls_first: null -> 0, valid -> 1 ; nulls_last: null -> 1, valid -> 0   (not affected by desc)
    return valid ? (c.nulls_first ? 1u : 0u) : (c.nulls_first ? 0u : 1u);
  }
  if (!valid) return 0;
  const int vb = b - c.has_null_byte;  // byte inside the value part
  if (c.dtype == B2_STRING) {
    const int32_t s = c.offsets[row], len = c.offsets[row + 1] - s;
    if (vb < c.str_max) out = vb < len ? reinterpret_cast<const uint8_t*>(c.data)[s + vb] : 0u;
    else out = ((uint32_t)len >> (8 * (3 - (vb - c.str_max)))) & 255u;  // 4-byte big-endian length tiebreak
  } else if (c.width == 16) {
    const uint64_t* p = reinterpret_cast<const uint64_t*>(c.data) + 2 * row;
    uint64_t hi = p[1] ^ 0x8000000000000000ull, lo = p[0];
    out = vb < 8 ? (uint32_t)(hi >> (8 * (7 - vb))) & 255u : (uint32_t)(lo >> (8 * (15 - vb))) & 255u;
  } else {
    uint64_t u;
    switch (c.dtype) {
      case B2_FLOAT32: {
        float f = reinterpret_cast<const float*>(c.data)[row];
        uint32_t x = (f != f) ? 0x7fc00000u : (f == 0.0f ? 0u : __float_as_uint(f));
        x = (x & 0x80000000u) ? ~x : (x | 0x80000000u);
        u = x;
      } break;
      case B2_FLOAT64: {
        double d = reinterpret_cast<const double*>(c.data)[row];
        uint64_t x = (d != d) ? 0x7ff8000000000000ull : (d == 0.0 ? 0ull : (uint64_t)__double_as_longlong(d));
        u = (x & 0x8000000000000000ull) ? ~x : (x | 0x8000000000000000ull);
      } break;
      default:
        switch (c.width) {
          case 1: u = (uint8_t)(reinterpret_cast<const uint8_t*>(c.data)[row] ^ 0x80u); break;
          case 2: u = (uint16_t)(reinterpret_cast<const uint16_t*>(c.data)[row] ^ 0x8000u); break;
          case 4: u = reinterpret_cast<const uint32_t*>(c.data)[row] ^ 0x80000000u; break;
          default: u = reinterpret_cast<const uint64_t*>(c.data)[row] ^ 0x8000000000000000ull; break;
        }
    }
    out = (uint32_t)(u >> (8 * (c.width - 1 - vb))) & 255u;
  }
  return c.ascending ? out : (out ^ 255u);
}

// bytes [8*chunk, 8*chunk+8) of the row key of `row` (byte 8*chunk most significant)
__device__ __forceinline__ uint64_t key_chunk(const SortPlan& plan, int64_t row, int chunk) {
  uint64_t k = 0;
  const int b0 = chunk * 8;
  for (int ci = 0; ci < plan.ncols; ci++) {
    const SortCol& c = plan.c[ci];
    const int lo = max(b0, c.key_off), hi = min(b0 + 8, c.key_off + c.key_len);
    for (int b = lo; b < hi; b++) k |= (uint64_t)norm_byte(c, row, b - c.key_off) << (8 * (7 - (b - b0)));
  }
  return k;
}

// keys[i] = chunk `chunk` of the row key of row perm[i]
__global__ void build_chunk_kernel(const __grid_constant__ SortPlan plan, const int32_t* __restrict__ perm, int64_t n, int chunk,
                                   uint64_t* __restrict__ keys) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    keys[i] = key_chunk(plan, perm ? perm[i] : i, chunk);
}

__global__ void max_strlen_kernel(const int32_t* __restrict__ offsets, int64_t n, int32_t* out) {
  int32_t m = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    m = max(m, offsets[i + 1] - offsets[i]);
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// str_max (optional, one entry per key): the padded length of each string key, for plans that must line up with the plans of
// other tables; otherwise the longest string of the column
SortPlan make_sort_plan(const Table* t, const b2_order_by_arg* keys, int nkeys, bool force_null_byte = false, const int32_t* str_max = nullptr) {
  B2_CHECK(nkeys >= 1 && nkeys <= SORT_MAX_KEYS, "bad number of sort keys");
  SortPlan p; memset(&p, 0, sizeof(p));
  p.ncols = nkeys;
  int off = 0;
  for (int k = 0; k < nkeys; k++) {
    B2_CHECK(keys[k].column >= 0 && keys[k].column < (int)t->cols.size(), "sort key column out of range");
    const Column* col = t->cols[keys[k].column];
    SortCol& c = p.c[k];
    c.data = col->data.p; c.valid = col->validity(); c.offsets = col->offsets.as<int32_t>();
    c.dtype = col->dtype; c.width = dtype_width(col->dtype);
    c.ascending = keys[k].ascending; c.nulls_first = keys[k].nulls_first;
    c.has_null_byte = (col->nullable() || force_null_byte) ? 1 : 0;
    int vlen = c.width;
    if (col->dtype == B2_STRING && str_max) {
      c.str_max = str_max[k];
      vlen = c.str_max + 4;
    } else if (col->dtype == B2_STRING) {
      DevBuf m(4);
      CUDA_CHECK(cudaMemsetAsync(m.p, 0, 4, stream()));
      if (col->size) launch(max_strlen_kernel, grid_for(col->size, 256), 256, 0, stream(), col->offsets.as<int32_t>(), col->size, m.as<int32_t>());
      int32_t mx = 0;
      d2h(&mx, m.p, 1);
      sync();
      if (mx > 1024) throw Error(B2_ERR_UNSUPPORTED, "sort keys over strings longer than 1024 bytes");
      c.str_max = mx;
      vlen = mx + 4;
    }
    c.key_off = off; c.key_len = vlen + c.has_null_byte;
    off += c.key_len;
  }
  p.key_bytes = off;
  return p;
}

// Small inputs (the candidates of a top-N, a final merge of per-rank top-Ns): ONE CTA sorts row indices in shared memory with a
// bitonic network over the normalised key chunks, ties broken by the row index (= the stable order).  The radix path costs
// ~5 launches per non-trivial digit — ~35 launches for the 8 K candidates of TPC-H q3's top-10 — whatever n is.
constexpr int SS_MAX = 16384, SS_NT = 1024;
__global__ void __launch_bounds__(SS_NT) small_sort_kernel(const uint64_t* __restrict__ keys, int nchunks, int n, int npow2, int32_t* __restrict__ perm_out) {
  extern __shared__ int32_t s_perm[];   // npow2 row indices; indices >= n are padding and sort behind every row
  for (int i = threadIdx.x; i < npow2; i += SS_NT) s_perm[i] = i;
  __syncthreads();
  auto less = [&](int a, int b) {
    if (a < n && b < n)
      for (int c = 0; c < nchunks; c++) {
        const uint64_t x = keys[(size_t)c * n + a], y = keys[(size_t)c * n + b];
        if (x != y) return x < y;
      }
    return a < b;
  };
  for (int k = 2; k <= npow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < npow2; i += SS_NT) {
        const int l = i ^ j;
        if (l > i) {
          const int a = s_perm[i], b = s_perm[l];
          const bool up = (i & k) == 0;
          if (less(b, a) == up) { s_perm[i] = b; s_perm[l] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < n; i += SS_NT) perm_out[i] = s_perm[i];
}

// stable argsort -> device int32 permutation (DevBuf of n ints)
DevBuf sort_order(const Table* t, const b2_order_by_arg* keys, int nkeys) {
  const int64_t n = t->rows;
  SortPlan plan = make_sort_plan(t, keys, nkeys);
  DevBuf perm_a((size_t)std::max<int64_t>(n, 1) * 4), perm_b((size_t)std::max<int64_t>(n, 1) * 4);
  if (n == 0) return perm_a;
  launch(iota32_kernel, grid_for(n, 256), 256, 0, stream(), perm_a.as<int32_t>(), n);
  if (n == 1) return perm_a;
  const int nchunks = (plan.key_bytes + 7) / 8;
  if (n <= SS_MAX && !getenv("B2_SORT_NO_SMALL")) {
    DevBuf kk((size_t)nchunks * n * 8);
    for (int chunk = 0; chunk < nchunks; chunk++)
      launch(build_chunk_kernel, grid_for(n, 256), 256, 0, stream(), plan, nullptr, n, chunk, kk.as<uint64_t>() + (size_t)chunk * n);
    int npow2 = 2;
    while (npow2 < n) npow2 <<= 1;
    const int smem = npow2 * 4;
    launch("small_sort_kernel", small_sort_kernel, 1, SS_NT, smem, stream(), kk.as<uint64_t>(), nchunks, (int)n, npow2, perm_a.as<int32_t>());
    return perm_a;
  }
  DevBuf keys_a((size_t)n * 8), keys_b((size_t)n * 8);
  bool in_a = true;
  for (int chunk = nchunks - 1; chunk >= 0; chunk--) {
    int32_t* pin = in_a ? perm_a.as<int32_t>() : perm_b.as<int32_t>();
    int32_t* pout = in_a ? perm_b.as<int32_t>() : perm_a.as<int32_t>();
    launch(build_chunk_kernel, grid_for(n, 256), 256, 0, stream(), plan, pin, n, chunk, keys_a.as<uint64_t>());
    // the low (8 - used) bytes of the last chunk are zero and get skipped as trivial digits
    int r = radix_sort_pairs(keys_a.as<uint64_t>(), pin, keys_b.as<uint64_t>(), pout, n, 8);
    if (r == 1) in_a = !in_a;
  }
  return in_a ? std::move(perm_a) : std::move(perm_b);
}

// ------------------------------------------------------------------------------------------------
// lower / upper bound of each `values` row in the sorted table (Table.lowerBound / upperBound,
// SortUtils.scala:172-203; GpuRangePartitioner.scala:187-196)
__global__ void bounds_kernel(const __grid_constant__ SortPlan sorted, const __grid_constant__ SortPlan vals, int64_t nsorted, int64_t nvals,
                              int upper, int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvals; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = nsorted;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      // compare sorted[mid] with vals[i] on normalised bytes (both plans carry a null byte per column)
      int cmp = 0;
      for (int ci = 0; ci < sorted.ncols && cmp == 0; ci++) {
        const SortCol& a = sorted.c[ci];
        const SortCol& b = vals.c[ci];
        for (int k = 0; k < a.key_len && cmp == 0; k++) {
          const uint32_t x = norm_byte(a, mid, k), y = norm_byte(b, i, k);
          cmp = x < y ? -1 : (x > y ? 1 : 0);
        }
      }
      const bool go_right = upper ? (cmp <= 0) : (cmp < 0);
      if (go_right) lo = mid + 1; else hi = mid;
    }
    out[i] = (int32_t)lo;
  }
}

Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols);
Table* concat_tables(const std::vector<const Table*>& ts);
Table* filter_by_mask(const Table* t, Column* m);

// plans of several tables whose normalised keys line up byte for byte: every key column has a null byte and each string key
// the padding of the longest string over all the tables (bounds_kernel compares two such plans)
std::vector<SortPlan> shared_sort_plans(const std::vector<const Table*>& ts, const b2_order_by_arg* keys, int nkeys) {
  std::vector<int32_t> str_max(std::max(nkeys, 1), 0);
  for (const Table* t : ts) {
    SortPlan p = make_sort_plan(t, keys, nkeys, true);
    for (int k = 0; k < nkeys; k++) str_max[k] = std::max(str_max[k], p.c[k].str_max);
  }
  std::vector<SortPlan> out;
  for (const Table* t : ts) out.push_back(make_sort_plan(t, keys, nkeys, true, str_max.data()));
  return out;
}

// the first row of `sorted` that does not sort before row 0 of `probe` (both tables hold the key columns `keys` refers to)
int64_t lower_bound_row(const Table* sorted, const Table* probe, const b2_order_by_arg* keys, int nkeys) {
  B2_CHECK(probe->rows >= 1, "bounds: empty probe");
  std::vector<SortPlan> p = shared_sort_plans({sorted, probe}, keys, nkeys);
  DevBuf out(4);
  launch(bounds_kernel, 1, 32, 0, stream(), p[0], p[1], sorted->rows, 1, 0, out.as<int32_t>());
  int32_t h = 0;
  d2h(&h, out.p, 1);
  sync();
  return h;
}

// ------------------------------------------------------------------------------------------------
// Merge of sorted runs (Table.merge, SortUtils.scala:249-301): a tree of pairwise merge-path merges of adjacent runs over the
// runs' concatenation, producing one gather map.  Rows are compared by the first 8-byte chunk of their normalised key, kept
// next to the map (8 B per row whatever the key width); only rows whose first chunks are equal compute their further chunks
// from the columns (key_chunk, the sort's own definition of the order).  On equal keys the left run wins: stable.
constexpr int MP_NT = 256, MP_ITEMS = 8, MP_TILE = MP_NT * MP_ITEMS;

struct MergeRuns {
  const uint64_t* keys; const int32_t* rows;   // run A = [a0, a0 + na), run B = [a0 + na, a0 + na + nb) of these arrays
  int64_t a0, na, nb;
  uint64_t* keys_out; int32_t* rows_out;       // output [a0, a0 + na + nb); keys_out null on the last level
};

// tie (optional): a per-row INT64 the caller orders by after the keys (the out-of-core sort's input position), read directly
// instead of through the normalised key
__device__ __forceinline__ bool mp_less(const SortPlan& plan, int nchunks, const int64_t* tie, uint64_t ka, int32_t ra, uint64_t kb, int32_t rb) {
  if (ka != kb) return ka < kb;
  for (int c = 1; c < nchunks; c++) {
    const uint64_t x = key_chunk(plan, ra, c), y = key_chunk(plan, rb, c);
    if (x != y) return x < y;
  }
  return tie && tie[ra] < tie[rb];
}

// number of A rows among the first `d` outputs: the largest i with A[i-1] <= B[d-i] (A wins ties)
template <typename KA, typename RA>
__device__ __forceinline__ int64_t mp_search(const SortPlan& plan, int nchunks, const int64_t* tie, KA ak, RA ar, int64_t na, KA bk, RA br, int64_t nb,
                                             int64_t d) {
  int64_t lo = max((int64_t)0, d - nb), hi = min(d, na);
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (!mp_less(plan, nchunks, tie, bk[d - 1 - mid], br[d - 1 - mid], ak[mid], ar[mid])) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// split[t] = A rows before output tile t (t = 0 .. ntiles)
__global__ void merge_path_partition_kernel(const __grid_constant__ SortPlan plan, int nchunks, const int64_t* __restrict__ tie, MergeRuns m, int64_t ntiles, int64_t* __restrict__ split) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t > ntiles) return;
  const int64_t d = min(t * MP_TILE, m.na + m.nb);
  const uint64_t* ak = m.keys + m.a0; const int32_t* ar = m.rows + m.a0;
  split[t] = mp_search(plan, nchunks, tie, ak, ar, m.na, ak + m.na, ar + m.na, m.nb, d);
}

// aligned 16-byte vector stores of the destination for the n elements src[idx[0..n)] in shared memory (scalar head and tail)
template <typename T>
__device__ __forceinline__ void mp_store(T* __restrict__ dst, const T* src, const uint16_t* idx, int n) {
  constexpr int V = 16 / sizeof(T);
  int head = (int)(((16 - ((uintptr_t)dst & 15)) & 15) / sizeof(T));
  if (head > n) head = n;
  for (int i = threadIdx.x; i < head; i += MP_NT) dst[i] = src[idx[i]];
  const int nvec = (n - head) / V;
  uint4* dv = reinterpret_cast<uint4*>(dst + head);
  for (int v = threadIdx.x; v < nvec; v += MP_NT) {
    union { uint4 u; T e[V]; } w;
#pragma unroll
    for (int k = 0; k < V; k++) w.e[k] = src[idx[head + v * V + k]];
    dv[v] = w.u;
  }
  for (int i = head + nvec * V + threadIdx.x; i < n; i += MP_NT) dst[i] = src[idx[i]];
}

// one CTA per output tile: stage the tile's A and B ranges in shared memory (loads issued in batches of MP_ITEMS per lane),
// each thread merges MP_ITEMS outputs found by its own merge-path search and notes where each output's row is staged; the
// tile then leaves as aligned vectors
__global__ void __launch_bounds__(MP_NT) merge_path_kernel(const __grid_constant__ SortPlan plan, int nchunks, const int64_t* __restrict__ tie, MergeRuns m,
                                                           const int64_t* __restrict__ split) {
  __shared__ __align__(16) uint64_t s_key[MP_TILE];
  __shared__ __align__(16) int32_t s_row[MP_TILE];
  __shared__ uint16_t s_src[MP_TILE];
  const int64_t t = blockIdx.x, n = m.na + m.nb;
  const int64_t d0 = t * MP_TILE, d1 = min(d0 + MP_TILE, n);
  const int64_t a_lo = split[t], a_hi = split[t + 1];
  const int64_t b_lo = d0 - a_lo, b_hi = d1 - a_hi;
  const int na = (int)(a_hi - a_lo), nb = (int)(b_hi - b_lo), cnt = na + nb;
  {
    uint64_t k[MP_ITEMS]; int32_t r[MP_ITEMS];
#pragma unroll
    for (int i = 0; i < MP_ITEMS; i++) {
      const int s = i * MP_NT + threadIdx.x;
      const int64_t g = s < na ? m.a0 + a_lo + s : m.a0 + m.na + b_lo + (s - na);
      if (s < cnt) { k[i] = m.keys[g]; r[i] = m.rows[g]; }
    }
#pragma unroll
    for (int i = 0; i < MP_ITEMS; i++) {
      const int s = i * MP_NT + threadIdx.x;
      if (s < cnt) { s_key[s] = k[i]; s_row[s] = r[i]; }
    }
  }
  __syncthreads();
  const int diag = min((int)threadIdx.x * MP_ITEMS, cnt);
  int i = (int)mp_search(plan, nchunks, tie, s_key, s_row, na, s_key + na, s_row + na, nb, diag);
  int j = diag - i;
#pragma unroll
  for (int q = 0; q < MP_ITEMS; q++) {   // s_src[output] = staged position of its row
    const bool take_a = j >= nb || (i < na && !mp_less(plan, nchunks, tie, s_key[na + j], s_row[na + j], s_key[i], s_row[i]));
    const int o = diag + q;
    if (o < cnt) s_src[o] = (uint16_t)(take_a ? i : na + j);
    if (take_a) i++; else j++;
  }
  __syncthreads();
  mp_store(m.rows_out + m.a0 + d0, s_row, s_src, cnt);
  if (m.keys_out) mp_store(m.keys_out + m.a0 + d0, s_key, s_src, cnt);
}

// gather map (int32, t->rows entries) that merges the sorted runs [off[r], off[r+1]) of `t`; rows with equal keys are
// ordered by tie[row] when `tie` is given (device, t->rows entries), else by run
DevBuf merge_runs(const Table* t, const std::vector<int64_t>& off, const b2_order_by_arg* keys, int nkeys, const int64_t* tie) {
  const int64_t n = t->rows;
  B2_CHECK(!off.empty() && off.front() == 0 && off.back() == n, "merge: run offsets do not cover the table");
  if (n > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "merge of more than 2^31-1 rows");
  DevBuf rows_a((size_t)std::max<int64_t>(n, 1) * 4);
  if (n) launch(iota32_kernel, grid_for(n, 256), 256, 0, stream(), rows_a.as<int32_t>(), n);
  std::vector<int64_t> runs;   // boundaries of the non-empty runs
  for (size_t r = 0; r + 1 < off.size(); r++) {
    B2_CHECK(off[r + 1] >= off[r], "merge: run offsets decrease");
    if (off[r + 1] > off[r]) runs.push_back(off[r]);
  }
  runs.push_back(n);
  const SortPlan plan = make_sort_plan(t, keys, nkeys, true);   // also checks the keys when there is nothing to merge
  if (runs.size() <= 2) return rows_a;
  const int nchunks = (plan.key_bytes + 7) / 8;
  DevBuf keys_a((size_t)n * 8), keys_b((size_t)n * 8), rows_b((size_t)n * 4);
  launch(build_chunk_kernel, grid_for(n, 256), 256, 0, stream(), plan, nullptr, n, 0, keys_a.as<uint64_t>());
  DevBuf split((size_t)((n + MP_TILE - 1) / MP_TILE + 2) * 8);
  while (runs.size() > 2) {
    const bool last = runs.size() == 3;
    std::vector<int64_t> next;
    for (size_t r = 0; r + 1 < runs.size(); r += 2) {
      next.push_back(runs[r]);
      if (r + 2 >= runs.size()) {   // odd run out: carried to the next level unchanged
        const size_t len = (size_t)(runs[r + 1] - runs[r]);
        CUDA_CHECK(cudaMemcpyAsync(rows_b.as<int32_t>() + runs[r], rows_a.as<int32_t>() + runs[r], len * 4, cudaMemcpyDeviceToDevice, stream()));
        CUDA_CHECK(cudaMemcpyAsync(keys_b.as<uint64_t>() + runs[r], keys_a.as<uint64_t>() + runs[r], len * 8, cudaMemcpyDeviceToDevice, stream()));
        continue;
      }
      MergeRuns m{keys_a.as<uint64_t>(), rows_a.as<int32_t>(), runs[r], runs[r + 1] - runs[r], runs[r + 2] - runs[r + 1],
                  last ? nullptr : keys_b.as<uint64_t>(), rows_b.as<int32_t>()};
      const int64_t ntiles = (m.na + m.nb + MP_TILE - 1) / MP_TILE;
      launch("merge_path_partition_kernel", merge_path_partition_kernel, (int)((ntiles + 1 + 127) / 128), 128, 0, stream(), plan, nchunks, tie, m,
             ntiles, split.as<int64_t>());
      launch("merge_path_kernel", merge_path_kernel, (int)ntiles, MP_NT, 0, stream(), plan, nchunks, tie, m, split.as<int64_t>());
    }
    next.push_back(n);
    runs.swap(next);
    std::swap(rows_a, rows_b);
    std::swap(keys_a, keys_b);
  }
  return rows_a;
}

// histogram of digit (key >> shift) & 255 over the rows whose key agrees with `pval` on the bits of `pmask`
__global__ void __launch_bounds__(256) hist_prefix_kernel(const uint64_t* __restrict__ keys, int64_t n, uint64_t pmask, uint64_t pval, int shift,
                                                          unsigned long long* __restrict__ hist) {
  __shared__ uint32_t s_h[256];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t k = keys[i];
    if ((k & pmask) == pval) atomicAdd(&s_h[(k >> shift) & 255], 1u);
  }
  __syncthreads();
  if (s_h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long)s_h[threadIdx.x]);
}

__global__ void topn_mask_kernel(const uint64_t* __restrict__ keys, int64_t n, uint64_t thr, int8_t* __restrict__ mask) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) mask[i] = keys[i] <= thr;
}

// Top-N without sorting the batch: radix-select on the most significant varying byte of the row key.  One histogram
// pass over the leading 8 key bytes gives the smallest byte value b whose cumulative count reaches the limit; every
// row of the answer has a key prefix <= b, so the batch is compacted (in input order: ties stay stable) to those
// candidates and only they are sorted.  Returns nullptr when the prefix does not discriminate (caller sorts).
static Table* top_n_select(const Table* t, const b2_order_by_arg* keys, int nkeys, int64_t limit) {
  const int64_t n = t->rows;
  if (n < (1 << 18) || limit <= 0 || limit > n / 16) return nullptr;
  SortPlan plan = make_sort_plan(t, keys, nkeys);
  DevBuf k0((size_t)n * 8);
  DevBuf hist(8 * 256 * 8);
  const int nchunks = (plan.key_bytes + 7) / 8;
  uint64_t thr = 0;
  int64_t m = -1;
  // leading 8-byte chunks of the row key on which ALL rows agree cannot discriminate (e.g. the high half of a DECIMAL128
  // revenue): the selection moves on to the next chunk, every row still being a candidate
  for (int chunk = 0; chunk < nchunks && m < 0; chunk++) {
    launch(build_chunk_kernel, grid_for(n, 256), 256, 0, stream(), plan, nullptr, n, chunk, k0.as<uint64_t>());
    CUDA_CHECK(cudaMemsetAsync(hist.p, 0, hist.bytes, stream()));
    launch(hist8_kernel, grid_for(n, 256 * 8), 256, 0, stream(), k0.as<uint64_t>(), n, 8, hist.as<unsigned long long>());
    std::vector<unsigned long long> h(8 * 256);
    d2h(h.data(), hist.p, h.size());
    sync();
    thr = 0;
    int d = 7;
    for (; d >= 0; d--) {   // leading digits of this chunk on which all rows agree
      int constant = -1;
      for (int b = 0; b < 256; b++) if (h[d * 256 + b] == (unsigned long long)n) constant = b;
      if (constant < 0) break;
      thr |= (uint64_t)constant << (8 * d);
    }
    if (d < 0) continue;   // the whole chunk is constant: the next chunk decides
    // radix select from the first varying digit down: each round histograms the next digit of the rows that still tie with
    // the prefix, keeps the bucket in which the limit-th smallest key lies and stops once few rows share the prefix
    int64_t k = limit, below = 0;
    uint64_t pmask = d == 7 ? 0 : ~((1ull << (8 * (d + 1))) - 1);
    uint64_t pval = thr;
    std::vector<unsigned long long> hd(h.begin() + d * 256, h.begin() + (d + 1) * 256);
    while (true) {
      int64_t cum = 0; int b = 0;
      for (; b < 256; b++) { if (cum + (int64_t)hd[b] >= k) break; cum += (int64_t)hd[b]; }
      below += cum; k -= cum;
      pval |= (uint64_t)b << (8 * d); pmask |= 0xffull << (8 * d);
      const int64_t tied = (int64_t)hd[b];
      if (d == 0 || tied <= 8192) { thr = pval | (d > 0 ? (1ull << (8 * d)) - 1 : 0); m = below + tied; break; }
      d--;
      CUDA_CHECK(cudaMemsetAsync(hist.p, 0, 256 * 8, stream()));
      launch(hist_prefix_kernel, grid_for(n, 256 * 8), 256, 0, stream(), k0.as<uint64_t>(), n, pmask, pval, 8 * d, hist.as<unsigned long long>());
      d2h(hd.data(), hist.p, 256);
      sync();
    }
  }
  if (m < 0 || m > n / 4) return nullptr;   // all leading bytes equal, or one value dominates: sort everything
  ColGuard mask(new_column(B2_BOOL8, 0, n, false));
  launch(topn_mask_kernel, grid_for(n, 256), 256, 0, stream(), k0.as<uint64_t>(), n, thr, mask.c->data.as<int8_t>());
  std::unique_ptr<Table, void (*)(Table*)> sub(filter_by_mask(t, mask.c), table_release);
  if (sub->rows < std::min<int64_t>(limit, n)) throw Error(B2_ERR_INVALID, "top-n selection lost rows");
  DevBuf perm = sort_order(sub.get(), keys, nkeys);
  return gather_table(sub.get(), perm.as<int32_t>(), std::min<int64_t>(limit, sub->rows), false, nullptr);
}


// GpuTopN (limit.scala:234-330): the first `limit` rows of the sorted batch — radix select when it pays, else a full sort
Table* top_n_table(const Table* t, const b2_order_by_arg* keys, int nkeys, int64_t limit) {
  if (Table* sel = top_n_select(t, keys, nkeys, limit)) return sel;
  DevBuf perm = sort_order(t, keys, nkeys);
  return gather_table(t, perm.as<int32_t>(), std::min<int64_t>(limit, t->rows), false, nullptr);
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_sort_order(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys, b2_handle* out_int32_perm) {
  B2_TRY
  Table* t = table_from(table);
  DevBuf perm = sort_order(t, keys, nkeys);
  std::unique_ptr<Column> c(new Column());
  c->dtype = B2_INT32; c->size = t->rows; c->data = std::move(perm);
  *out_int32_perm = to_handle(c.release());
  B2_CATCH
}

int b2_order_by(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys, b2_handle* out_table) {
  B2_TRY
  Table* t = table_from(table);
  DevBuf perm = sort_order(t, keys, nkeys);
  *out_table = to_handle(gather_table(t, perm.as<int32_t>(), t->rows, false, nullptr));
  B2_CATCH
}

int b2_top_n(b2_handle table, const b2_order_by_arg* keys, int32_t nkeys, int64_t n, b2_handle* out_table) {
  B2_TRY
  // GpuTopN (limit.scala:234-330): the first n rows of the sorted batch
  Table* t = table_from(table);
  B2_CHECK(n >= 0, "negative limit");
  *out_table = to_handle(top_n_table(t, keys, nkeys, n));
  B2_CATCH
}

int b2_merge_sorted(const b2_handle* tables, int32_t ntables, const b2_order_by_arg* keys, int32_t nkeys, b2_handle* out_table) {
  B2_TRY
  // Table.merge (SortUtils.scala:301): the inputs are sorted; the merge-path tree over their concatenation keeps equal keys
  // in input-table order, as the stable sort of the concatenation would
  B2_CHECK(ntables >= 1, "merge of zero tables");
  std::vector<const Table*> ts;
  std::vector<int64_t> off{0};
  for (int i = 0; i < ntables; i++) { ts.push_back(table_from(tables[i])); off.push_back(off.back() + ts.back()->rows); }
  std::unique_ptr<Table, void (*)(Table*)> cat(concat_tables(ts), table_release);
  DevBuf perm = merge_runs(cat.get(), off, keys, nkeys, nullptr);
  *out_table = to_handle(gather_table(cat.get(), perm.as<int32_t>(), cat->rows, false, nullptr));
  B2_CATCH
}

int b2_search_bounds(b2_handle sorted_table, b2_handle values_table, const b2_order_by_arg* keys, int32_t nkeys, int32_t upper,
                     b2_handle* out_int32_idx) {
  B2_TRY
  Table* st = table_from(sorted_table);
  Table* vt = table_from(values_table);
  // both tables hold exactly the key columns, in key order
  std::vector<b2_order_by_arg> k(keys, keys + nkeys);
  for (int i = 0; i < nkeys; i++) k[i].column = i;
  B2_CHECK((int)st->cols.size() >= nkeys && (int)vt->cols.size() >= nkeys, "bounds tables must hold the key columns");
  for (int i = 0; i < nkeys; i++) {
    B2_CHECK(st->cols[i]->dtype == vt->cols[i]->dtype, "bounds: key dtypes differ");
    if (st->cols[i]->dtype == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "bounds search over string keys");
  }
  SortPlan sp = make_sort_plan(st, k.data(), nkeys, true), vp = make_sort_plan(vt, k.data(), nkeys, true);
  ColGuard out(new_column(B2_INT32, 0, vt->rows, false));
  if (vt->rows) launch(bounds_kernel, grid_for(vt->rows, 128), 128, 0, stream(), sp, vp, st->rows, vt->rows, upper, out.c->data.as<int32_t>());
  *out_int32_idx = to_handle(out.release());
  B2_CATCH
}

}  // extern "C"
