// rows.cu — a11: columnar <-> JCUDF fixed-width rows (RowConversion.convertToRowsFixedWidthOptimized /
// convertFromRows; GpuColumnarToRowExec.scala:44-220, 386-400; GpuRowToColumnarExec.scala:574-755).
// Layout (shims/CudfUnsafeRowBase.scala:80-90, 234-246): every column at an offset aligned to its
// own width, then ceil(ncols/8) validity bytes (bit i of byte i/8 set = column i valid), row size
// rounded up to 8 bytes.
//
// Both directions stage a tile of rows in shared memory so that the column side is read/written
// one-thread-per-row (coalesced per column) and the row side is moved as contiguous 16-byte words.
#include "common.cuh"

namespace b2 {

constexpr int RW_MAX_COLS = 64;
struct RowLayout {
  int32_t ncols;
  int32_t row_bytes;
  int32_t validity_off;
  int32_t off[RW_MAX_COLS];
  int32_t width[RW_MAX_COLS];
  void* data[RW_MAX_COLS];
  uint32_t* valid[RW_MAX_COLS];
};

static RowLayout layout_for(const int32_t* dtypes, int ncols) {
  if (ncols < 1 || ncols > RW_MAX_COLS) throw Error(B2_ERR_UNSUPPORTED, "row conversion supports 1..64 columns");
  RowLayout L; memset(&L, 0, sizeof(L));
  L.ncols = ncols;
  int off = 0;
  for (int c = 0; c < ncols; c++) {
    if (dtypes[c] == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "fixed-width row conversion does not take strings");
    int w = dtype_width(dtypes[c]);
    off = (off + w - 1) & -w;
    L.off[c] = off; L.width[c] = w;
    off += w;
  }
  L.validity_off = off;
  L.row_bytes = (off + (ncols + 7) / 8 + 7) & ~7;
  if (L.row_bytes > 1536) throw Error(B2_ERR_UNSUPPORTED, "row wider than 1.5 KB");  // GpuColumnarToRowExec.scala:123-134
  return L;
}

__global__ void __launch_bounds__(256) to_rows_kernel(const __grid_constant__ RowLayout L, int64_t nrows, int rows_per_tile, uint8_t* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t tile[];
  const int64_t ntiles = (nrows + rows_per_tile - 1) / rows_per_tile;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t base = t * rows_per_tile;
    const int here = (int)min((long long)rows_per_tile, (long long)(nrows - base));
    for (int k = threadIdx.x; k < here * L.row_bytes / 4; k += blockDim.x) reinterpret_cast<uint32_t*>(tile)[k] = 0;
    __syncthreads();
    for (int r = threadIdx.x; r < here; r += blockDim.x) {
      uint8_t* row = tile + (size_t)r * L.row_bytes;
      const int64_t g = base + r;
      for (int c = 0; c < L.ncols; c++) {
        const bool v = row_valid(L.valid[c], g);
        if (v) row[L.validity_off + (c >> 3)] |= (uint8_t)(1u << (c & 7));
        switch (L.width[c]) {
          case 1: *(row + L.off[c]) = reinterpret_cast<const uint8_t*>(L.data[c])[g]; break;
          case 2: *reinterpret_cast<uint16_t*>(row + L.off[c]) = reinterpret_cast<const uint16_t*>(L.data[c])[g]; break;
          case 4: *reinterpret_cast<uint32_t*>(row + L.off[c]) = reinterpret_cast<const uint32_t*>(L.data[c])[g]; break;
          case 8: *reinterpret_cast<uint64_t*>(row + L.off[c]) = reinterpret_cast<const uint64_t*>(L.data[c])[g]; break;
          default: {  // rows are only 8-byte aligned in shared memory
            const ulonglong2 v16 = reinterpret_cast<const ulonglong2*>(L.data[c])[g];
            reinterpret_cast<uint64_t*>(row + L.off[c])[0] = v16.x; reinterpret_cast<uint64_t*>(row + L.off[c])[1] = v16.y;
          } break;
        }
      }
    }
    __syncthreads();
    const uint64_t* src = reinterpret_cast<const uint64_t*>(tile);
    uint64_t* dst = reinterpret_cast<uint64_t*>(out + base * L.row_bytes);
    for (int k = threadIdx.x; k < here * L.row_bytes / 8; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) from_rows_kernel(const __grid_constant__ RowLayout L, int64_t nrows, int rows_per_tile, const uint8_t* __restrict__ in) {
  extern __shared__ __align__(16) uint8_t tile[];
  const int64_t ntiles = (nrows + rows_per_tile - 1) / rows_per_tile;  // rows_per_tile is a multiple of 32
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t base = t * rows_per_tile;
    const int here = (int)min((long long)rows_per_tile, (long long)(nrows - base));
    const uint64_t* src = reinterpret_cast<const uint64_t*>(in + base * L.row_bytes);
    uint64_t* dst = reinterpret_cast<uint64_t*>(tile);
    for (int k = threadIdx.x; k < here * L.row_bytes / 8; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
    const int rounded = (here + 31) & ~31;
    for (int r = threadIdx.x; r < rounded; r += blockDim.x) {
      const bool in_range = r < here;
      const uint8_t* row = tile + (size_t)r * L.row_bytes;
      const int64_t g = base + r;
      for (int c = 0; c < L.ncols; c++) {
        bool v = false;
        if (in_range) {
          v = (row[L.validity_off + (c >> 3)] >> (c & 7)) & 1;
          switch (L.width[c]) {
            case 1: reinterpret_cast<uint8_t*>(L.data[c])[g] = *(row + L.off[c]); break;
            case 2: reinterpret_cast<uint16_t*>(L.data[c])[g] = *reinterpret_cast<const uint16_t*>(row + L.off[c]); break;
            case 4: reinterpret_cast<uint32_t*>(L.data[c])[g] = *reinterpret_cast<const uint32_t*>(row + L.off[c]); break;
            case 8: reinterpret_cast<uint64_t*>(L.data[c])[g] = *reinterpret_cast<const uint64_t*>(row + L.off[c]); break;
            default: {
              ulonglong2 v16;
              v16.x = reinterpret_cast<const uint64_t*>(row + L.off[c])[0]; v16.y = reinterpret_cast<const uint64_t*>(row + L.off[c])[1];
              reinterpret_cast<ulonglong2*>(L.data[c])[g] = v16;
            } break;
          }
        }
        const uint32_t bits = __ballot_sync(0xffffffffu, v);
        if ((threadIdx.x & 31) == 0 && in_range) L.valid[c][g >> 5] = bits;
      }
    }
    __syncthreads();
  }
}

static int pick_rows_per_tile(int row_bytes) {
  int r = (96 * 1024) / row_bytes;
  r &= ~31;
  if (r > 1024) r = 1024;
  if (r < 32) r = 32;
  return r;
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_rows_size(b2_handle table, int32_t* row_bytes) {
  B2_TRY
  Table* t = table_from(table);
  std::vector<int32_t> dts;
  for (auto* c : t->cols) dts.push_back(c->dtype);
  *row_bytes = layout_for(dts.data(), (int)dts.size()).row_bytes;
  B2_CATCH
}

int b2_table_to_rows(b2_handle table, uint8_t* host_rows, int64_t capacity_bytes) {
  B2_TRY
  Table* t = table_from(table);
  std::vector<int32_t> dts;
  for (auto* c : t->cols) dts.push_back(c->dtype);
  RowLayout L = layout_for(dts.data(), (int)dts.size());
  const int64_t total = t->rows * L.row_bytes;
  B2_CHECK(capacity_bytes >= total, "row buffer too small");
  if (total > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "row batch exceeds 2 GiB; split the batch");
  if (t->rows == 0) return B2_OK;
  for (size_t c = 0; c < t->cols.size(); c++) { L.data[c] = t->cols[c]->data.p; L.valid[c] = t->cols[c]->valid.as<uint32_t>(); }
  DevBuf rows((size_t)total);
  const int rpt = pick_rows_per_tile(L.row_bytes);
  launch(to_rows_kernel, grid_for(t->rows, rpt, 2), 256, rpt * L.row_bytes, stream(), L, t->rows, rpt, rows.as<uint8_t>());
  CUDA_CHECK(cudaMemcpyAsync(host_rows, rows.p, (size_t)total, cudaMemcpyDeviceToHost, stream()));
  sync();
  B2_CATCH
}

int b2_table_from_rows(const uint8_t* host_rows, int64_t nrows, const int32_t* dtypes, const int32_t* scales, int32_t ncols, b2_handle* out_table) {
  B2_TRY
  RowLayout L = layout_for(dtypes, ncols);
  ColsGuard outs;
  for (int c = 0; c < ncols; c++) {
    Column* col = new_column(dtypes[c], scales ? scales[c] : 0, nrows, true);
    outs.v.push_back(col);
    L.data[c] = col->data.p; L.valid[c] = col->valid.as<uint32_t>();
  }
  if (nrows) {
    const int64_t total = nrows * L.row_bytes;
    DevBuf rows((size_t)total);
    CUDA_CHECK(cudaMemcpyAsync(rows.p, host_rows, (size_t)total, cudaMemcpyHostToDevice, stream()));
    const int rpt = pick_rows_per_tile(L.row_bytes);
    launch(from_rows_kernel, grid_for(nrows, rpt, 2), 256, rpt * L.row_bytes, stream(), L, nrows, rpt, rows.as<uint8_t>());
    sync();
  }
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

}  // extern "C"
