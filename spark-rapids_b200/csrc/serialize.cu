// serialize.cu — (f1) the shuffle wire format: host-side serialised tables and coalesce-on-read.
// Reference: GpuColumnarBatchSerializer.scala:169-320 (serialize a batch / a row slice to the shuffle stream as
// "header + host buffer"), :385-470 (deserialize to SerializedTableColumn), GpuShuffleCoalesceExec.scala:72-110, 371-475
// (read N serialised tables, concatenate them ON THE HOST up to the batch target, then ONE host->device copy).
// The byte format the reference writes is cudf-java's JCudfSerialization / spark-rapids-jni's Kudo; neither source is in
// /root/reference, so bit compatibility cannot be established here.  This file defines an equivalent self-describing
// format ("B2T1": fixed header, per-column descriptors, then validity / offsets / data buffers each padded to 64 bytes —
// the same structure as JCudfSerialization's header + contiguous host buffer) and implements the same three operations:
// serialise a row range of a device table into host memory, size it, and concatenate serialised tables into one device
// table with a single upload per column.  oracle/shuffle_format.py is the independent reader that pins the layout.
//
//   SerHeader { u32 magic 'B2T1'; u16 version = 1; u16 ncols; i64 rows; i64 total_bytes }              24 bytes
//   SerCol[ncols] { i32 dtype; i32 scale; i64 null_count; i64 validity_bytes; i64 offsets_bytes; i64 data_bytes }   40 bytes each
//   padding to 64, then for every column: validity (LSB-first bits, absent when null_count == 0; the reader ignores the
//   bits past the last row) | offsets (int32, rebased to 0, STRING only) | data — each padded to a multiple of 64 bytes.
#include <algorithm>
#include <deque>
#include "common.cuh"

namespace b2 {

Table* slice_table(const Table* t, int64_t start, int64_t end);

constexpr uint32_t SER_MAGIC = 0x31543242u;  // "B2T1" little endian
struct SerHeader { uint32_t magic; uint16_t version, ncols; int64_t rows, total_bytes; };
struct SerCol { int32_t dtype, scale; int64_t null_count, validity_bytes, offsets_bytes, data_bytes; };
static_assert(sizeof(SerHeader) == 24 && sizeof(SerCol) == 40, "wire structs are packed as documented");
static inline int64_t pad64i(int64_t b) { return (b + 63) & ~(int64_t)63; }

struct SerPlan { std::vector<SerCol> cols; int64_t payload_off = 0, total = 0; };
static SerPlan plan_of(const Table* t) {   // t is already the slice to write
  SerPlan p;
  for (auto* c : t->cols) {
    SerCol sc; memset(&sc, 0, sizeof(sc));
    sc.dtype = c->dtype; sc.scale = c->scale;
    sc.null_count = c->null_count;   // finalised by the caller
    sc.validity_bytes = sc.null_count > 0 ? (t->rows + 7) / 8 : 0;
    sc.offsets_bytes = c->dtype == B2_STRING ? (t->rows + 1) * 4 : 0;
    sc.data_bytes = c->dtype == B2_STRING ? c->chars_bytes : t->rows * dtype_width(c->dtype);
    p.cols.push_back(sc);
  }
  p.payload_off = pad64i((int64_t)sizeof(SerHeader) + (int64_t)p.cols.size() * (int64_t)sizeof(SerCol));
  p.total = p.payload_off;
  for (auto& sc : p.cols) p.total += pad64i(sc.validity_bytes) + pad64i(sc.offsets_bytes) + pad64i(sc.data_bytes);
  return p;
}

struct TableHold { Table* t = nullptr; ~TableHold() { if (t) table_release(t); } };

// the rows [start, end) of t as a table whose buffers can be copied out verbatim (offsets rebased, validity from bit 0)
static Table* slice_for_wire(Table* t, int64_t start, int64_t end) {
  if (start == 0 && end == t->rows) { t->refs.fetch_add(1); return t; }
  return slice_table(t, start, end);
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_serialized_size(b2_handle table, int64_t row_start, int64_t row_end, int64_t* out_bytes) {
  B2_TRY
  Table* t = table_from(table);
  B2_CHECK(row_start >= 0 && row_end >= row_start && row_end <= t->rows, "row range out of bounds");
  TableHold h; h.t = slice_for_wire(t, row_start, row_end);
  for (auto* c : h.t->cols) finalize_nulls(c);
  *out_bytes = plan_of(h.t).total;
  B2_CATCH
}

// GpuColumnarBatchSerializer: one serialised table per (batch, partition slice)
int b2_serialize_table(b2_handle table, int64_t row_start, int64_t row_end, uint8_t* host_out, int64_t capacity, int64_t* out_written) {
  B2_TRY
  Table* t = table_from(table);
  B2_CHECK(row_start >= 0 && row_end >= row_start && row_end <= t->rows, "row range out of bounds");
  B2_CHECK((int)t->cols.size() <= 0xffff, "too many columns");
  TableHold h; h.t = slice_for_wire(t, row_start, row_end);
  for (auto* c : h.t->cols) finalize_nulls(c);
  SerPlan p = plan_of(h.t);
  B2_CHECK(capacity >= p.total, "serialisation buffer too small (b2_serialized_size)");
  memset(host_out, 0, (size_t)p.payload_off);
  SerHeader hd; hd.magic = SER_MAGIC; hd.version = 1; hd.ncols = (uint16_t)h.t->cols.size(); hd.rows = h.t->rows; hd.total_bytes = p.total;
  memcpy(host_out, &hd, sizeof(hd));
  memcpy(host_out + sizeof(hd), p.cols.data(), p.cols.size() * sizeof(SerCol));
  int64_t off = p.payload_off;
  cudaStream_t s = stream();
  for (size_t i = 0; i < p.cols.size(); i++) {
    const SerCol& sc = p.cols[i];
    const Column* c = h.t->cols[i];
    auto put = [&](const void* dev, int64_t bytes) {
      if (bytes) CUDA_CHECK(cudaMemcpyAsync(host_out + off, dev, (size_t)bytes, cudaMemcpyDeviceToHost, s));
      const int64_t padded = pad64i(bytes);
      if (padded > bytes) memset(host_out + off + bytes, 0, (size_t)(padded - bytes));
      off += padded;
    };
    put(c->valid.p, sc.validity_bytes);
    put(c->offsets.p, sc.offsets_bytes);
    put(c->data.p, sc.data_bytes);
  }
  sync();
  *out_written = p.total;
  B2_CATCH
}

// A descriptor must agree with its table's row count, and its buffers must lie inside the serialised table: the reader
// copies by row count, so a descriptor that declares fewer bytes than its rows need would make it read past the buffer.
// String offsets must start at 0, never decrease and end at data_bytes; set bits must number rows - null_count.
static void check_column(const uint8_t* buf, const SerHeader& h, const SerCol& sc, int64_t cur) {
  const int64_t n = h.rows;
  const bool str = sc.dtype == B2_STRING;
  B2_CHECK(sc.dtype >= B2_BOOL8 && sc.dtype <= B2_STRING, "serialised column has an unknown type");
  B2_CHECK(sc.null_count >= 0 && sc.null_count <= n, "serialised column: null_count out of range");
  B2_CHECK(sc.validity_bytes == (sc.null_count > 0 ? (n + 7) / 8 : 0), "serialised column: validity_bytes disagrees with rows / null_count");
  B2_CHECK(sc.offsets_bytes == (str ? (n + 1) * 4 : 0), "serialised column: offsets_bytes disagrees with rows");
  B2_CHECK(str ? sc.data_bytes >= 0 : sc.data_bytes == n * dtype_width(sc.dtype), "serialised column: data_bytes disagrees with rows");
  B2_CHECK(sc.data_bytes <= h.total_bytes && cur + pad64i(sc.validity_bytes) + pad64i(sc.offsets_bytes) + pad64i(sc.data_bytes) <= h.total_bytes,
           "serialised table is truncated");
  if (sc.validity_bytes) {
    const uint8_t* v = buf + cur;
    int64_t set = 0;
    for (int64_t k = 0; k < n / 8; k++) set += __builtin_popcount(v[k]);
    if (n & 7) set += __builtin_popcount(v[n / 8] & ((1u << (n & 7)) - 1u));
    B2_CHECK(set == n - sc.null_count, "serialised column: null_count disagrees with the validity bits");
  }
  if (str) {
    const int32_t* o = reinterpret_cast<const int32_t*>(buf + cur + pad64i(sc.validity_bytes));
    B2_CHECK(o[0] == 0 && o[n] == sc.data_bytes, "serialised string offsets must run from 0 to data_bytes");
    for (int64_t r = 0; r < n; r++) B2_CHECK(o[r] <= o[r + 1], "serialised string offsets decrease");
  }
}

// GpuShuffleCoalesceExec: N serialised tables -> ONE device table; the concatenation happens on the host (validity bits
// shifted into place, string offsets rebased), then each column buffer is uploaded once.
int b2_deserialize_concat(const uint8_t* const* bufs, const int64_t* lens, int32_t nbufs, b2_handle* out_table) {
  B2_TRY
  B2_CHECK(nbufs >= 1, "nothing to deserialise");
  std::vector<const SerHeader*> hs;
  std::vector<const SerCol*> cs;
  int64_t rows = 0;
  for (int b = 0; b < nbufs; b++) {
    B2_CHECK(lens[b] >= (int64_t)sizeof(SerHeader), "serialised table is truncated");
    const SerHeader* h = reinterpret_cast<const SerHeader*>(bufs[b]);
    B2_CHECK(h->magic == SER_MAGIC && h->version == 1, "not a B2T1 serialised table");
    B2_CHECK(h->ncols == reinterpret_cast<const SerHeader*>(bufs[0])->ncols, "serialised tables differ in column count");
    B2_CHECK(h->total_bytes <= lens[b] && h->total_bytes >= pad64i((int64_t)sizeof(SerHeader) + (int64_t)h->ncols * (int64_t)sizeof(SerCol)) &&
             h->rows >= 0 && h->rows <= 0x7fffffffLL, "serialised table is truncated");
    hs.push_back(h);
    cs.push_back(reinterpret_cast<const SerCol*>(bufs[b] + sizeof(SerHeader)));
    rows += h->rows;
  }
  if (rows > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "coalesced shuffle batch exceeds 2^31-1 rows");
  const int ncols = hs[0]->ncols;
  // running payload cursor of every input
  std::vector<int64_t> cur(nbufs);
  for (int b = 0; b < nbufs; b++) cur[b] = pad64i((int64_t)sizeof(SerHeader) + (int64_t)ncols * (int64_t)sizeof(SerCol));
  ColsGuard outs;
  cudaStream_t s = stream();
  std::deque<std::vector<uint8_t>> staging;   // host concatenations stay alive until the copies are done (deque: references stay valid)
  for (int i = 0; i < ncols; i++) {
    const int dtype = cs[0][i].dtype;
    int64_t nulls = 0, chars = 0;
    for (int b = 0; b < nbufs; b++) {
      B2_CHECK(cs[b][i].dtype == dtype && cs[b][i].scale == cs[0][i].scale, "serialised tables differ in column type");
      check_column(bufs[b], *hs[b], cs[b][i], cur[b]);
      nulls += cs[b][i].null_count; chars += cs[b][i].data_bytes;
    }
    if (dtype == B2_STRING && chars > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "coalesced string column exceeds 2^31-1 chars");
    std::unique_ptr<Column> oc(new Column());
    oc->dtype = dtype; oc->scale = cs[0][i].scale; oc->size = rows; oc->null_count = nulls;
    const int w = dtype == B2_STRING ? 0 : dtype_width(dtype);
    staging.emplace_back(); std::vector<uint8_t>& vbuf = staging.back();
    staging.emplace_back(); std::vector<uint8_t>& obuf = staging.back();
    staging.emplace_back(); std::vector<uint8_t>& dbuf = staging.back();
    if (nulls > 0) vbuf.assign(validity_bytes(rows), 0);
    if (dtype == B2_STRING) obuf.resize((size_t)(rows + 1) * 4);
    dbuf.resize((size_t)(dtype == B2_STRING ? chars : rows * w));
    int64_t row = 0, ch = 0;
    for (int b = 0; b < nbufs; b++) {
      const SerCol& sc = cs[b][i];
      const int64_t n = hs[b]->rows;
      const uint8_t* v = bufs[b] + cur[b]; cur[b] += pad64i(sc.validity_bytes);
      const uint8_t* o = bufs[b] + cur[b]; cur[b] += pad64i(sc.offsets_bytes);
      const uint8_t* d = bufs[b] + cur[b]; cur[b] += pad64i(sc.data_bytes);
      if (nulls > 0) {
        if (sc.validity_bytes == 0) { for (int64_t r = 0; r < n; r++) vbuf[(size_t)((row + r) >> 3)] |= (uint8_t)(1u << ((row + r) & 7)); }
        else if ((row & 7) == 0) {
          uint8_t* dst = vbuf.data() + (row >> 3);
          memcpy(dst, v, (size_t)((n + 7) / 8));
          // the writer need not zero the bits past its last row: they would mark the next input's first rows valid
          if (n & 7) dst[n >> 3] &= (uint8_t)((1u << (n & 7)) - 1u);
        }
        else for (int64_t r = 0; r < n; r++) if ((v[r >> 3] >> (r & 7)) & 1) vbuf[(size_t)((row + r) >> 3)] |= (uint8_t)(1u << ((row + r) & 7));
      }
      if (dtype == B2_STRING) {
        const int32_t* so = reinterpret_cast<const int32_t*>(o);
        int32_t* dst = reinterpret_cast<int32_t*>(obuf.data()) + row;
        for (int64_t r = 0; r < n; r++) dst[r] = so[r] + (int32_t)ch;
        if (sc.data_bytes) memcpy(dbuf.data() + ch, d, (size_t)sc.data_bytes);
        ch += sc.data_bytes;
      } else if (n) memcpy(dbuf.data() + row * w, d, (size_t)(n * w));
      row += n;
    }
    if (dtype == B2_STRING) {
      reinterpret_cast<int32_t*>(obuf.data())[rows] = (int32_t)ch;
      oc->offsets = DevBuf(obuf.size());
      CUDA_CHECK(cudaMemcpyAsync(oc->offsets.p, obuf.data(), obuf.size(), cudaMemcpyHostToDevice, s));
      oc->chars_bytes = ch;
    }
    oc->data = DevBuf(dbuf.size());
    if (!dbuf.empty()) CUDA_CHECK(cudaMemcpyAsync(oc->data.p, dbuf.data(), dbuf.size(), cudaMemcpyHostToDevice, s));
    if (nulls > 0) {
      oc->valid = DevBuf(vbuf.size());
      CUDA_CHECK(cudaMemcpyAsync(oc->valid.p, vbuf.data(), vbuf.size(), cudaMemcpyHostToDevice, s));
    }
    outs.v.push_back(oc.release());
  }
  sync();   // the staging vectors go away on return
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

}  // extern "C"
