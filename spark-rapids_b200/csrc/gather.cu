// gather.cu — a7 (Table.gather(map, OutOfBoundsPolicy), JoinGatherer.scala:585-599), a12
// (Table.concatenate, GpuAggregateExec.scala:700-727 / GpuCoalesceBatches.scala:43-108) and slicing
// (contiguousSplit pieces, GpuPartitioning.scala:66-99).
//
// The reference launches one cudf gather per column; here one kernel reads the int32 map once per
// output row and moves every fixed-width payload column for that row (fused payload gather), with
// validity assembled by warp ballot.  Strings take a size pass + scan + copy pass.
#include "prim.cuh"

namespace b2 {

constexpr int G_MAX_COLS = 64;
struct GatherCols {
  int32_t ncols;
  int32_t width[G_MAX_COLS];
  const void* in[G_MAX_COLS];
  const uint32_t* in_valid[G_MAX_COLS];
  void* out[G_MAX_COLS];
  uint32_t* out_valid[G_MAX_COLS];
};

template <typename T>
__device__ __forceinline__ void gather_one(const void* in, void* out, int64_t i, int32_t m, bool ok) {
  reinterpret_cast<T*>(out)[i] = ok ? reinterpret_cast<const T*>(in)[m] : T();
}

__global__ void __launch_bounds__(256) gather_fixed_kernel(const __grid_constant__ GatherCols gc, const int32_t* __restrict__ map,
                                                           int64_t n, int64_t src_rows) {
  const int64_t nround = (n + 31) & ~(int64_t)31;  // whole warps so that ballots are complete
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
    const bool in_range = i < n;
    int32_t m = in_range ? map[i] : -1;
    const bool ok = in_range && m >= 0 && m < src_rows;
    for (int c = 0; c < gc.ncols; c++) {
      if (in_range) {
        switch (gc.width[c]) {
          case 1: gather_one<int8_t>(gc.in[c], gc.out[c], i, m, ok); break;
          case 2: gather_one<int16_t>(gc.in[c], gc.out[c], i, m, ok); break;
          case 4: gather_one<int32_t>(gc.in[c], gc.out[c], i, m, ok); break;
          case 8: gather_one<int64_t>(gc.in[c], gc.out[c], i, m, ok); break;
          case 16: gather_one<longlong2>(gc.in[c], gc.out[c], i, m, ok); break;
          default: break;
        }
      }
      if (gc.out_valid[c]) {
        bool v = ok && row_valid(gc.in_valid[c], m);
        uint32_t bits = __ballot_sync(0xffffffffu, v);
        if ((threadIdx.x & 31) == 0 && in_range) gc.out_valid[c][i >> 5] = bits;
      }
    }
  }
}

__global__ void string_sizes_kernel(const int32_t* __restrict__ offsets, const int32_t* __restrict__ map, int64_t n, int64_t src_rows,
                                    const uint32_t* __restrict__ in_valid, int32_t* __restrict__ sizes, uint32_t* __restrict__ out_valid) {
  const int64_t nround = (n + 31) & ~(int64_t)31;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
    bool in_range = i < n;
    int32_t m = in_range ? map[i] : -1;
    bool ok = in_range && m >= 0 && m < src_rows;
    bool v = ok && row_valid(in_valid, m);
    if (in_range) sizes[i] = v ? offsets[m + 1] - offsets[m] : 0;
    if (out_valid) {
      uint32_t bits = __ballot_sync(0xffffffffu, v);
      if ((threadIdx.x & 31) == 0 && in_range) out_valid[i >> 5] = bits;
    }
  }
}

// one warp per output string
__global__ void string_copy_kernel(const int32_t* __restrict__ in_off, const uint8_t* __restrict__ in_chars,
                                   const int32_t* __restrict__ map, int64_t n, int64_t src_rows,
                                   const int32_t* __restrict__ out_off, uint8_t* __restrict__ out_chars) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    const int32_t o0 = out_off[i], len = out_off[i + 1] - o0;
    if (len == 0) continue;
    const int32_t m = map[i];
    const uint8_t* src = in_chars + in_off[m];
    for (int k = lane; k < len; k += 32) out_chars[o0 + k] = src[k];
  }
}

__global__ void iota_kernel(int32_t* out, int64_t n, int32_t start) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = start + (int32_t)i;
}

static Column* gather_string(const Column* ic, const int32_t* d_map, int64_t n, bool nullable_out) {
  std::unique_ptr<Column> oc(new Column());
  oc->dtype = B2_STRING; oc->size = n;
  oc->offsets = DevBuf((size_t)(n + 1) * 4);
  if (nullable_out) { oc->valid = DevBuf(validity_bytes(n)); oc->null_count = -1; }
  if (n == 0) {
    CUDA_CHECK(cudaMemsetAsync(oc->offsets.p, 0, 4, stream()));
    oc->data = DevBuf(0);
    return oc.release();
  }
  launch(string_sizes_kernel, grid_for(n, 256), 256, 0, stream(), ic->offsets.as<int32_t>(), d_map, n, ic->size, ic->validity(),
         oc->offsets.as<int32_t>(), oc->valid.as<uint32_t>());
  DevBuf sums = exclusive_scan<int32_t, int32_t>(oc->offsets.as<int32_t>(), oc->offsets.as<int32_t>(), n, true);
  int64_t total = 0;
  int64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  d2h(&total, sums.as<int64_t>() + ntiles, 1);
  sync();
  if (total > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "gathered string column exceeds 2^31-1 chars");
  oc->chars_bytes = total;
  oc->data = DevBuf((size_t)total);
  if (total)
    launch(string_copy_kernel, grid_for(n * 32, 256), 256, 0, stream(), ic->offsets.as<int32_t>(), ic->data.as<uint8_t>(), d_map, n, ic->size,
           oc->offsets.as<int32_t>(), oc->data.as<uint8_t>());
  return oc.release();
}

// gather rows of `t` by a device int32 map.  OOB (incl. negative) index -> NULL row when
// nullify_oob (OutOfBoundsPolicy.NULLIFY), else the map must be in range (DONT_CHECK).
Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols) {
  std::vector<int> cols;
  if (only_cols) cols = *only_cols;
  else for (int c = 0; c < (int)t->cols.size(); c++) cols.push_back(c);
  if (n > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "gather output exceeds 2^31-1 rows");
  ColsGuard outs;
  outs.v.resize(cols.size(), nullptr);
  GatherCols gc; memset(&gc, 0, sizeof(gc));
  std::vector<int> fixed_slots;
  auto flush = [&]() {
    if (gc.ncols == 0 || n == 0) { gc.ncols = 0; return; }
    launch("gather_fixed_kernel", gather_fixed_kernel, grid_for(n, 256), 256, 0, stream(), gc, d_map, n, t->rows);
    gc.ncols = 0;
  };
  for (size_t k = 0; k < cols.size(); k++) {
    const Column* ic = t->cols[cols[k]];
    bool nullable_out = ic->nullable() || nullify_oob;
    if (ic->dtype == B2_STRING) { outs.v[k] = gather_string(ic, d_map, n, nullable_out); continue; }
    Column* oc = new_column(ic->dtype, ic->scale, n, nullable_out);
    outs.v[k] = oc;
    int s = gc.ncols++;
    gc.width[s] = dtype_width(ic->dtype);
    gc.in[s] = ic->data.p; gc.in_valid[s] = ic->validity();
    gc.out[s] = oc->data.p; gc.out_valid[s] = oc->valid.as<uint32_t>();
    if (gc.ncols == G_MAX_COLS) flush();
  }
  flush();
  return new_table(outs.release());
}

// ------------------------------------------------------------------------------------------------
__global__ void copy_bits_kernel(const uint32_t* __restrict__ src, int64_t src_start, uint32_t* __restrict__ dst, int64_t dst_start,
                                 int64_t n) {
  // sets bits [dst_start, dst_start+n) of dst from src (src may be null = all valid); dst pre-zeroed
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool v = src == nullptr || bit_get(src, src_start + i);
    if (v) atomicOr(&dst[(dst_start + i) >> 5], 1u << ((dst_start + i) & 31));
  }
}
__global__ void rebase_offsets_kernel(const int32_t* __restrict__ src, int64_t n, int32_t delta, int32_t* __restrict__ dst) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[i] + delta;
}

Table* concat_tables(const std::vector<const Table*>& ts) {
  B2_CHECK(!ts.empty(), "concat of zero tables");
  size_t ncols = ts[0]->cols.size();
  int64_t total = 0;
  for (auto* t : ts) {
    B2_CHECK(t->cols.size() == ncols, "concat: column count differs");
    total += t->rows;
  }
  if (total > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "concatenated table exceeds 2^31-1 rows");
  ColsGuard outs;
  for (size_t c = 0; c < ncols; c++) {
    const Column* c0 = ts[0]->cols[c];
    bool any_null = false;
    for (auto* t : ts) {
      B2_CHECK(t->cols[c]->dtype == c0->dtype, "concat: dtype differs");
      B2_CHECK(!is_decimal(c0->dtype) || t->cols[c]->scale == c0->scale, "concat: decimal scale differs");
      any_null = any_null || t->cols[c]->nullable();
    }
    if (c0->dtype == B2_STRING) {
      int64_t chars = 0;
      for (auto* t : ts) chars += t->cols[c]->chars_bytes;
      if (chars > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "concatenated string column exceeds 2^31-1 chars");
      std::unique_ptr<Column> oc(new Column());
      oc->dtype = B2_STRING; oc->size = total; oc->chars_bytes = chars;
      oc->offsets = DevBuf((size_t)(total + 1) * 4);
      oc->data = DevBuf((size_t)chars);
      int64_t row = 0, ch = 0;
      for (auto* t : ts) {
        const Column* ic = t->cols[c];
        if (ic->size) {
          launch(rebase_offsets_kernel, grid_for(ic->size, 256), 256, 0, stream(), ic->offsets.as<int32_t>(), ic->size, (int32_t)ch,
                 oc->offsets.as<int32_t>() + row);
          if (ic->chars_bytes)
            CUDA_CHECK(cudaMemcpyAsync(oc->data.as<char>() + ch, ic->data.p, (size_t)ic->chars_bytes, cudaMemcpyDeviceToDevice, stream()));
        }
        row += ic->size; ch += ic->chars_bytes;
      }
      int32_t last = (int32_t)chars;
      h2d(oc->offsets.as<int32_t>() + total, &last, 1);
      sync();
      outs.v.push_back(oc.release());
    } else {
      Column* oc = new_column(c0->dtype, c0->scale, total, any_null);
      outs.v.push_back(oc);
      int w = dtype_width(c0->dtype);
      int64_t row = 0;
      for (auto* t : ts) {
        const Column* ic = t->cols[c];
        if (ic->size)
          CUDA_CHECK(cudaMemcpyAsync(oc->data.as<char>() + row * w, ic->data.p, (size_t)ic->size * w, cudaMemcpyDeviceToDevice, stream()));
        row += ic->size;
      }
    }
    if (any_null) {
      Column* oc = outs.v.back();
      if (!oc->valid.p) oc->valid = DevBuf(validity_bytes(total));
      CUDA_CHECK(cudaMemsetAsync(oc->valid.p, 0, oc->valid.bytes, stream()));
      int64_t row = 0;
      for (auto* t : ts) {
        const Column* ic = t->cols[c];
        if (ic->size) launch(copy_bits_kernel, grid_for(ic->size, 256), 256, 0, stream(), ic->validity(), 0, oc->valid.as<uint32_t>(), row, ic->size);
        row += ic->size;
      }
      oc->null_count = -1;
    }
  }
  return new_table(outs.release());
}

// ---- GpuSubstring (stringFunctions.scala:524-620) with literal pos / len, materialised ------------------------------------------
__device__ __forceinline__ int sub_utf8_len(uint8_t lead) { return lead < 0x80 ? 1 : ((lead >> 5) == 6 ? 2 : ((lead >> 4) == 14 ? 3 : ((lead >> 3) == 30 ? 4 : 1))); }
// byte window [b0, b1) of string [p, p+n) for Spark's substringSQL(pos, len): code-point based, 1-based pos, negative pos
// counts from the end; start = pos < 0 ? pos + nchars : (pos > 0 ? pos - 1 : 0), end = clamp(start + len, 0, INT_MAX)
__device__ __forceinline__ void substring_window(const uint8_t* p, int n, int64_t pos, int64_t len, int& b0, int& b1) {
  int nchars = 0;
  for (int k = 0; k < n; k++) nchars += (p[k] & 0xc0) != 0x80;
  int64_t start = pos < 0 ? pos + nchars : (pos > 0 ? pos - 1 : 0);
  int64_t end = start + len;
  if (end < 0) end = 0;
  if (end > 0x7fffffffLL) end = 0x7fffffffLL;
  if (start < 0) start = 0;
  b0 = b1 = 0;
  if (start >= end || start >= nchars) return;
  int c = 0;
  while (b0 < n && c < start) { b0 += sub_utf8_len(p[b0]); c++; }
  b1 = b0;
  while (b1 < n && c < end) { b1 += sub_utf8_len(p[b1]); c++; }
  if (b1 > n) b1 = n;
}
__global__ void substring_sizes_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ chars, const uint32_t* __restrict__ valid, int64_t n,
                                       int64_t pos, int64_t len, int32_t* __restrict__ sizes, int32_t* __restrict__ starts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int b0 = 0, b1 = 0;
    if (row_valid(valid, i)) substring_window(chars + offsets[i], offsets[i + 1] - offsets[i], pos, len, b0, b1);
    sizes[i] = b1 - b0; starts[i] = offsets[i] + b0;
  }
}
__global__ void substring_copy_kernel(const uint8_t* __restrict__ chars, const int32_t* __restrict__ starts, const int32_t* __restrict__ out_off, int64_t n,
                                      uint8_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t o = out_off[i], l = out_off[i + 1] - o;
    const uint8_t* s = chars + starts[i];
    for (int k = 0; k < l; k++) out[o + k] = s[k];
  }
}
Column* substring_column(const Column* ic, int64_t pos, int64_t len) {
  if (ic->dtype != B2_STRING) throw Error(B2_ERR_INVALID, "substring needs a STRING column");
  const int64_t n = ic->size;
  std::unique_ptr<Column> oc(new Column());
  oc->dtype = B2_STRING; oc->size = n;
  oc->offsets = DevBuf((size_t)(n + 1) * 4);
  if (ic->nullable()) {   // NULL in, NULL out (NullIntolerant)
    oc->valid = DevBuf(validity_bytes(n)); oc->null_count = ic->null_count;
    CUDA_CHECK(cudaMemcpyAsync(oc->valid.p, ic->valid.p, validity_bytes(n), cudaMemcpyDeviceToDevice, stream()));
  }
  if (n == 0) { CUDA_CHECK(cudaMemsetAsync(oc->offsets.p, 0, 4, stream())); oc->data = DevBuf(0); return oc.release(); }
  DevBuf starts((size_t)n * 4);
  launch(substring_sizes_kernel, grid_for(n, 256), 256, 0, stream(), ic->offsets.as<int32_t>(), ic->data.as<uint8_t>(), ic->validity(), n, pos, len,
         oc->offsets.as<int32_t>(), starts.as<int32_t>());
  DevBuf sums = exclusive_scan<int32_t, int32_t>(oc->offsets.as<int32_t>(), oc->offsets.as<int32_t>(), n, true);
  int64_t total = 0;
  d2h(&total, sums.as<int64_t>() + (n + SCAN_TILE - 1) / SCAN_TILE, 1);
  sync();
  oc->chars_bytes = total;
  oc->data = DevBuf((size_t)total);
  if (total)
    launch(substring_copy_kernel, grid_for(n, 256), 256, 0, stream(), ic->data.as<uint8_t>(), starts.as<int32_t>(), oc->offsets.as<int32_t>(), n,
           oc->data.as<uint8_t>());
  sync();   // `starts` is freed on return
  return oc.release();
}

Table* slice_table(const Table* t, int64_t start, int64_t end) {
  B2_CHECK(start >= 0 && end >= start && end <= t->rows, "slice out of range");
  int64_t n = end - start;
  DevBuf map((size_t)std::max<int64_t>(n, 1) * 4);
  if (n) launch(iota_kernel, grid_for(n, 256), 256, 0, stream(), map.as<int32_t>(), n, (int32_t)start);
  return gather_table(t, map.as<int32_t>(), n, false, nullptr);
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_gather(b2_handle table, b2_handle int32_map, int32_t nullify_oob, b2_handle* out_table) {
  B2_TRY
  Table* t = table_from(table);
  Column* m = col_from(int32_map);
  B2_CHECK(m->dtype == B2_INT32, "gather map must be INT32");
  *out_table = to_handle(gather_table(t, m->data.as<int32_t>(), m->size, nullify_oob != 0, nullptr));
  B2_CATCH
}

int b2_substring(b2_handle string_column, int32_t pos, int32_t len, b2_handle* out_column) {
  B2_TRY
  *out_column = to_handle(substring_column(col_from(string_column), pos, len));
  B2_CATCH
}

int b2_concat(const b2_handle* tables, int32_t ntables, b2_handle* out_table) {
  B2_TRY
  std::vector<const Table*> ts;
  for (int i = 0; i < ntables; i++) ts.push_back(table_from(tables[i]));
  *out_table = to_handle(concat_tables(ts));
  B2_CATCH
}

int b2_slice(b2_handle table, int64_t start, int64_t end, b2_handle* out_table) {
  B2_TRY
  *out_table = to_handle(slice_table(table_from(table), start, end));
  B2_CATCH
}

}  // extern "C"
