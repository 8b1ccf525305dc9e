// exec.cu — host-side operator layer above the kernels: the C++ mirror of the reference's GpuExec
// nodes for the hot path (the reference's host side is Scala; no JVM exists in this image, so the
// compiled-language mirror is C++).  Contract copied from GpuExec.internalDoExecuteColumnar():
// RDD[ColumnarBatch] (GpuExec.scala:106,190,380): every node is a pull iterator of batches; metrics
// numOutputRows / numOutputBatches / opTime (GpuExec.scala:195-199, GpuMetrics.scala:49-62).
//
//   GpuBatchSource            the child RDD / scan output handed in by the caller
//   GpuParquetScanExec        GpuParquetScan.scala:3543-3600 (PartitionReader.next -> Table.readParquet)
//   GpuFilterExec             basicPhysicalOperators.scala:1238-1291
//   GpuProjectExec            basicPhysicalOperators.scala:755-884
//   GpuHashAggregateExec      GpuAggregateExec.scala:1942-2085; first pass per batch (:730-742) then
//                             GpuMergeAggregateIterator (:896-1018): concat partials + merge-aggregate
//   GpuShuffledHashJoinExec   GpuShuffledHashJoinExec.scala:228-385 + GpuHashJoin.doJoin (:2547-2628):
//                             build side coalesced to ONE batch, hash table built once, stream probed
//                             batch by batch, payload gathered
//   GpuSortExec / GpuTopN     GpuSortExec.scala:87-165 (each-batch | full), limit.scala:234-330
//   GpuCoalesceBatches        GpuCoalesceBatches.scala:160-239 (TargetSize goal by rows)
//   GpuShuffleExchangeExec    GpuShuffleExchangeExecBase.scala:384-536 with the NCCL all-to-all
#include <algorithm>
#include <chrono>
#include <cmath>
#include <deque>
#include "joinemit.cuh"
#include "vm.cuh"

namespace b2 {

Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols);
Table* concat_tables(const std::vector<const Table*>& ts);
Table* scan_aggregate(const Program* prog, bool has_pred, const Table* t, const int* key_outs, int nkeys, const b2_agg_spec* specs, int naggs);
Program* make_passthrough_program(const Table* t, const std::vector<int>& cols);
Table* filter_select(const Program* prog, const Table* t, const int32_t* keep, int nkeep);
Column* filter_row_ids(const Program* prog, const Table* t);
bool join_probe_pred(b2_handle ht, const Table* batch, int key_col, const Program* prog, Column** out_lm, Column** out_rm, int64_t* npass_out,
                     b2_handle tracker);   // join.cu
Table* filter_by_mask(const Table* t, Column* m);
Column* rows_with_passing_pair(const Column* left_map, const Column* pass, int64_t stream_rows, bool invert);

Table* slice_table(const Table* t, int64_t start, int64_t end);
std::vector<Table*> hash_split_table(const Table* t, const int32_t* d_sel, int64_t n, const int32_t* key_cols, int nkeys, uint32_t seed,
                                     int nparts, const std::vector<int>& keep);   // hash.cu

// RmmRapidsRetryIterator.withRetry (RmmRapidsRetryIterator.scala:65-203): an allocation failure first spills (core.cu does
// that inside the allocator) and surfaces as B2_ERR_OOM = GpuRetryOOM; the operator then makes everything spillable leave
// the device, waits for the stream and runs the attempt again.  After two retries the error is handed to the caller, which
// for joins and aggregates splits the input batch in halves and retries each (GpuSplitAndRetryOOM semantics,
// AbstractGpuJoinIterator.scala:235-250 for the join's 2^31 output limit).
template <typename F>
static auto with_retry(F&& attempt) -> decltype(attempt()) {
  for (int n = 0;; n++) {
    try {
      return attempt();
    } catch (const Error& e) {
      if (e.code != B2_ERR_OOM || n >= 2) throw;
      note_retry();
      spill_device(INT64_MAX);
      CUDA_CHECK(cudaStreamSynchronize(stream()));
    }
  }
}
static bool splittable(const Error& e) { return e.code == B2_ERR_OOM || e.code == B2_ERR_SIZE_OVERFLOW; }

struct TableRef {  // owning reference
  Table* t = nullptr;
  TableRef() {}
  explicit TableRef(Table* t_) : t(t_) {}
  TableRef(const TableRef&) = delete;
  TableRef& operator=(const TableRef&) = delete;
  TableRef(TableRef&& o) noexcept : t(o.t) { o.t = nullptr; }
  TableRef& operator=(TableRef&& o) noexcept { if (this != &o) { reset(); t = o.t; o.t = nullptr; } return *this; }
  ~TableRef() { reset(); }
  void reset() { if (t) table_release(t); t = nullptr; }
  Table* release() { Table* r = t; t = nullptr; return r; }
};

static Table* from_handle_owned(b2_handle h) { return h ? reinterpret_cast<Table*>((intptr_t)h) : nullptr; }

// A batch waiting in the spill store, with the facts about it that planning needs, so that planning never brings it back
struct SpillPiece {
  b2_handle sp = 0;
  int64_t rows = 0, bytes = 0;
  std::vector<int64_t> chars;    // per column: string bytes
  std::vector<char> nullable;    // per column: carries validity
  SpillPiece() {}
  SpillPiece(const SpillPiece&) = delete;
  SpillPiece(SpillPiece&& o) noexcept : sp(o.sp), rows(o.rows), bytes(o.bytes), chars(std::move(o.chars)), nullable(std::move(o.nullable)) { o.sp = 0; }
  SpillPiece& operator=(SpillPiece&& o) noexcept {
    if (this != &o) { close(); sp = o.sp; o.sp = 0; rows = o.rows; bytes = o.bytes; chars = std::move(o.chars); nullable = std::move(o.nullable); }
    return *this;
  }
  ~SpillPiece() { close(); }
  // registers `t` (the store takes its own reference)
  void hold(const Table* t) {
    rows = t->rows; bytes = table_bytes(t);
    for (const Column* c : t->cols) { chars.push_back(c->dtype == B2_STRING ? c->chars_bytes : 0); nullable.push_back(c->nullable()); }
    int rc = b2_spillable_create(to_handle(const_cast<Table*>(t)), &sp);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
  }
  void close() { if (sp) b2_spillable_close(sp); sp = 0; }
  Table* get() const {
    b2_handle h = 0;
    int rc = b2_spillable_get(sp, &h);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    return from_handle_owned(h);
  }
};

static std::vector<TableRef> owned(std::vector<Table*>&& ts) {
  std::vector<TableRef> out;
  for (Table* t : ts) out.emplace_back(t);
  return out;
}
// GpuBatchSubPartitioner, shared by the join's sub-partitioning and the aggregate's repartitioning: the rows of t (or the n rows
// d_sel names), columns `keep`, split by pmod(murmur3(keys, seed), nparts) into spill pieces; put(p, piece) for every non-empty p
template <typename Put>
static void split_pieces(const Table* t, const int32_t* d_sel, int64_t n, const std::vector<int>& keys, const std::vector<int>& keep, int seed,
                         int nparts, Put&& put) {
  std::vector<TableRef> parts = owned(with_retry([&] { return hash_split_table(t, d_sel, n, keys.data(), (int)keys.size(), (uint32_t)seed, nparts, keep); }));
  for (int p = 0; p < nparts; p++) {
    if (!parts[p].t) continue;
    SpillPiece s;
    s.hold(parts[p].t);
    put(p, std::move(s));
  }
}
// the pieces brought back and concatenated (a new reference to `empty` when there are none)
static Table* concat_pieces(const std::vector<SpillPiece>& ps, const Table* empty) {
  return with_retry([&]() -> Table* {
    if (ps.empty()) { Table* e = const_cast<Table*>(empty); e->refs.fetch_add(1); return e; }
    std::vector<TableRef> got;
    std::vector<const Table*> ts;
    for (auto& p : ps) { got.emplace_back(p.get()); ts.push_back(got.back().t); }
    if (ts.size() == 1) return got[0].release();
    return concat_tables(ts);
  });
}

struct GpuExec {
  std::atomic<int> refs{1};
  std::vector<GpuExec*> children;
  int64_t num_output_rows = 0, num_output_batches = 0, op_time_ns = 0;
  // device time of this node (CUDA events on the library stream around every next(), recorded while profiling is on):
  // total includes the children pulled from inside next(); self = total - children  (opTime of GpuMetrics.scala:49-62)
  struct Span { cudaEvent_t a, b; };
  std::vector<Span> spans, child_spans;
  virtual ~GpuExec() {
    for (auto& sp : spans) { cudaEventDestroy(sp.a); cudaEventDestroy(sp.b); }
    for (auto* c : children) c->release();
  }
  void release() { if (refs.fetch_sub(1) == 1) delete this; }
  void add_child(GpuExec* c) { c->refs.fetch_add(1); children.push_back(c); }
  virtual Table* do_next() = 0;  // nullptr when exhausted; returned table is owned by the caller
  static GpuExec*& current() { static thread_local GpuExec* cur = nullptr; return cur; }
  Table* next() {
    const bool prof = profile_enabled();
    Span sp{nullptr, nullptr};
    if (prof) { cudaEventCreate(&sp.a); cudaEventCreate(&sp.b); cudaEventRecord(sp.a, stream()); }
    GpuExec* parent = current();
    struct Restore { GpuExec* p; ~Restore() { current() = p; } } restore{parent};
    current() = this;
    auto t0 = std::chrono::steady_clock::now();
    Table* t = do_next();
    op_time_ns += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    if (prof) { cudaEventRecord(sp.b, stream()); spans.push_back(sp); if (parent) parent->child_spans.push_back(sp); }
    if (t) { num_output_rows += t->rows; num_output_batches++; }
    return t;
  }
  // run f() as if node `who` had done it (an operator fused into this one keeps its own line in the metrics)
  template <typename F>
  auto run_as(GpuExec* who, F&& f) -> decltype(f()) {
    if (!profile_enabled()) return f();
    Span sp{nullptr, nullptr};
    cudaEventCreate(&sp.a); cudaEventCreate(&sp.b); cudaEventRecord(sp.a, stream());
    struct Done { Span& sp; GpuExec* who; GpuExec* me; ~Done() { cudaEventRecord(sp.b, stream()); who->spans.push_back(sp); me->child_spans.push_back(sp); } } done{sp, who, this};
    return f();
  }
  static double span_ms(const std::vector<Span>& v) {
    double ms = 0;
    for (auto& sp : v) { float t = 0; cudaEventSynchronize(sp.b); if (cudaEventElapsedTime(&t, sp.a, sp.b) == cudaSuccess) ms += t; }
    return ms;
  }
};
static GpuExec* exec_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null exec handle");
  return reinterpret_cast<GpuExec*>((intptr_t)h);
}

struct GpuBatchSource : GpuExec {
  std::deque<Table*> q;
  ~GpuBatchSource() { for (auto* t : q) table_release(t); }
  Table* do_next() override {
    if (q.empty()) return nullptr;
    Table* t = q.front(); q.pop_front();
    return t;
  }
};

struct GpuParquetScanExec : GpuExec {
  struct Buf { const uint8_t* p; int64_t len; };
  std::deque<Buf> bufs;
  std::vector<std::string> names;
  Table* do_next() override {
    if (bufs.empty()) return nullptr;
    Buf b = bufs.front(); bufs.pop_front();
    std::vector<const char*> cn;
    for (auto& s : names) cn.push_back(s.c_str());
    b2_handle out = 0;
    int rc = b2_parquet_decode(b.p, b.len, cn.data(), (int)cn.size(), &out);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    return from_handle_owned(out);
  }
};

struct GpuFilterExec : GpuExec {
  b2_handle program;
  std::vector<int32_t> keep;   // non-empty: a column-pruning GpuProjectExec above the filter, fused (only these are compacted)
  Table* do_next() override {
    TableRef in(children[0]->next());
    if (!in.t) return nullptr;
    if (!keep.empty()) return filter_select(program_from(program), in.t, keep.data(), (int)keep.size());
    b2_handle out = 0;
    int rc = b2_filter(program, to_handle(in.t), &out);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    return from_handle_owned(out);
  }
};

// HostColumnarToGpu (HostColumnarToGpu.scala; GpuRowToColumnarExec.scala:937-998 for the row source): host columnar batches
// -> device batches.  The copy of batch k+1 runs on the copy stream while batch k is being consumed downstream
// (the reference keeps host buffers in flight the same way: GpuMultiFileReader.scala).
struct HostColumn { int32_t dtype, scale; int64_t rows; const void* data; const uint8_t* validity; const int32_t* offsets; };
struct GpuHostBatchSource : GpuExec {
  std::vector<std::vector<HostColumn>> batches;
  size_t next_batch = 0;
  struct InFlight { Table* t = nullptr; cudaEvent_t done = nullptr; };
  std::deque<InFlight> flight;
  cudaStream_t copy = nullptr;
  int depth = 2;
  ~GpuHostBatchSource() {
    for (auto& f : flight) { if (f.done) { cudaEventSynchronize(f.done); cudaEventDestroy(f.done); } if (f.t) table_release(f.t); }
    if (copy) cudaStreamDestroy(copy);
  }
  void issue() {
    const auto& b = batches[next_batch++];
    cudaStream_t s = stream();
    if (!copy) CUDA_CHECK(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    ColsGuard cols;
    for (const HostColumn& h : b) {
      std::unique_ptr<Column> c(new Column());
      c->dtype = h.dtype; c->scale = h.scale; c->size = h.rows;
      if (h.rows > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "host batch of more than 2^31-1 rows");
      if (h.dtype == B2_STRING) {
        c->offsets = DevBuf((size_t)(h.rows + 1) * 4);
        c->chars_bytes = h.rows ? h.offsets[h.rows] : 0;
        c->data = DevBuf((size_t)c->chars_bytes);
      } else c->data = DevBuf((size_t)h.rows * dtype_width(h.dtype));
      if (h.validity) { c->valid = DevBuf(validity_bytes(h.rows)); c->null_count = -1; }
      cols.v.push_back(c.release());
    }
    // the buffers were allocated in compute-stream order: the copy stream may touch them only after that point
    cudaEvent_t ready;
    CUDA_CHECK(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventRecord(ready, s));
    CUDA_CHECK(cudaStreamWaitEvent(copy, ready, 0));
    cudaEventDestroy(ready);
    for (size_t i = 0; i < b.size(); i++) {
      const HostColumn& h = b[i];
      Column* c = cols.v[i];
      if (h.dtype == B2_STRING) {
        if (h.rows) CUDA_CHECK(cudaMemcpyAsync(c->offsets.p, h.offsets, (size_t)(h.rows + 1) * 4, cudaMemcpyHostToDevice, copy));
        else CUDA_CHECK(cudaMemsetAsync(c->offsets.p, 0, 4, copy));
        if (c->chars_bytes) CUDA_CHECK(cudaMemcpyAsync(c->data.p, h.data, (size_t)c->chars_bytes, cudaMemcpyHostToDevice, copy));
      } else if (h.rows) {
        CUDA_CHECK(cudaMemcpyAsync(c->data.p, h.data, (size_t)h.rows * dtype_width(h.dtype), cudaMemcpyHostToDevice, copy));
      }
      if (h.validity) {
        CUDA_CHECK(cudaMemsetAsync(c->valid.p, 0, c->valid.bytes, copy));
        CUDA_CHECK(cudaMemcpyAsync(c->valid.p, h.validity, (size_t)((h.rows + 7) / 8), cudaMemcpyHostToDevice, copy));
      }
      h2d_bytes_total += (h.dtype == B2_STRING ? (int64_t)(h.rows + 1) * 4 + c->chars_bytes : h.rows * dtype_width(h.dtype)) + (h.validity ? (h.rows + 7) / 8 : 0);
    }
    InFlight f;
    f.t = new_table(cols.release());
    CUDA_CHECK(cudaEventCreateWithFlags(&f.done, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventRecord(f.done, copy));
    flight.push_back(f);
  }
  int64_t h2d_bytes_total = 0;
  Table* do_next() override {
    while ((int)flight.size() < depth && next_batch < batches.size()) issue();
    if (flight.empty()) return nullptr;
    InFlight f = flight.front(); flight.pop_front();
    CUDA_CHECK(cudaStreamWaitEvent(stream(), f.done, 0));   // the consumer's stream is ordered after the copy; the host does not block
    cudaEventDestroy(f.done);
    TableRef t(f.t);   // released if the next copy cannot be issued (an OOM under an allocation limit)
    if (next_batch < batches.size() && (int)flight.size() < depth) issue();
    return t.release();
  }
};
struct GpuProjectExec : GpuExec {
  b2_handle program;
  Table* do_next() override {
    TableRef in(children[0]->next());
    if (!in.t) return nullptr;
    b2_handle out = 0;
    int rc = b2_project(program, to_handle(in.t), &out);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    return from_handle_owned(out);
  }
};

// GpuExpandExec (GpuExpandExec.scala): every input batch is projected once per projection list and the results are stacked —
// the plan Spark uses for GROUPING SETS / ROLLUP / several COUNT(DISTINCT).  Output rows = rows x projections, projection-major.
struct GpuExpandExec : GpuExec {
  std::vector<b2_handle> projections;
  Table* do_next() override {
    TableRef in(children[0]->next());
    if (!in.t) return nullptr;
    std::vector<TableRef> parts;
    for (b2_handle p : projections) {
      b2_handle out = 0;
      int rc = b2_project(p, to_handle(in.t), &out);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      parts.emplace_back(from_handle_owned(out));
    }
    if (parts.size() == 1) return parts[0].release();
    std::vector<const Table*> ts;
    for (auto& p : parts) ts.push_back(p.t);
    return concat_tables(ts);
  }
};

// A partial decimal sum that overflowed is NULL although its group saw valid input (Spark's buffer (sum, isEmpty) with sum NULL
// and isEmpty false); a merge must then give NULL, whereas a NULL partial of an empty / all-NULL group is skipped.  Marks the
// first kind of row: flag[r] = sum[r] is NULL and (no count column, or count[r] > 0); *npoisoned counts them.
__global__ void poisoned_sums_kernel(const uint32_t* __restrict__ sum_valid, const int64_t* __restrict__ count, int64_t n, int8_t* __restrict__ flag,
                                     unsigned long long* __restrict__ npoisoned) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const bool p = !((sum_valid[r >> 5] >> (r & 31)) & 1u) && (count == nullptr || count[r] > 0);
    flag[r] = p;
    if (p) atomicAdd(npoisoned, 1ull);
  }
}
// clears the validity bit of every row whose merged flag (MAX of the partials' flags) is set
__global__ void clear_poisoned_kernel(uint32_t* __restrict__ valid, const int8_t* __restrict__ flag, int64_t n) {
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < (n + 31) >> 5; w += (int64_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
    for (int b = 0; b < 32 && w * 32 + b < n; b++) m |= (uint32_t)(flag[w * 32 + b] != 0) << b;
    valid[w] &= ~m;
  }
}

// aggregate modes as in Spark: Partial/Complete run the update aggregates on raw input, Final merges
// partial buffers (SUM of sums, SUM of counts, MIN of mins, MAX of maxes).  A partial buffer is the keys, one column per
// aggregate, then one INT64 count of valid inputs per decimal SUM (Spark's isEmpty, GpuDecimalSum).  Complete mode keeps
// that count between its own passes only, and only where a NULL partial sum may also mean an empty group.
struct GpuHashAggregateExec : GpuExec {
  Program* program = nullptr;  // pre-step projection (+ fused predicate as output 0) for update mode; null in merge mode
  int mode = B2_AGG_MODE_PARTIAL;
  bool has_pred = false, done = false;
  std::vector<int> keys;               // update: program outputs; merge: leading input columns
  std::vector<b2_agg_spec> aggs;       // update: columns = program outputs; merge: columns = input columns
  std::vector<int> counted;            // the decimal SUMs whose partials carry a count column, in column order

  static bool decimal_sum(const b2_agg_spec& s) { return s.kind == B2_AGG_SUM && (s.out_dtype == B2_DECIMAL64 || s.out_dtype == B2_DECIMAL128); }
  void init_counted() {
    for (int i = 0; i < (int)aggs.size(); i++) {
      if (!decimal_sum(aggs[i])) continue;
      // complete mode, keyed, NOT NULL input: every group of a partial saw a valid value, so a NULL sum is an overflow
      const int o = aggs[i].column + (has_pred ? 1 : 0);
      if (mode == B2_AGG_MODE_COMPLETE) B2_CHECK(o >= 0 && o < (int)program->out_nullable.size(), "aggregate input index out of range");
      const bool need = mode != B2_AGG_MODE_COMPLETE || keys.empty() || program->out_nullable[o];
      if (need) counted.push_back(i);
    }
  }
  std::vector<b2_agg_spec> update_specs() const {
    std::vector<b2_agg_spec> u = aggs;
    for (int i : counted) u.push_back(b2_agg_spec{B2_AGG_COUNT, aggs[i].column, B2_INT64, 0, 0});
    return u;
  }
  static std::vector<b2_agg_spec> merge_specs(const std::vector<b2_agg_spec>& a, int nkeys) {
    std::vector<b2_agg_spec> m = a;
    for (size_t i = 0; i < m.size(); i++) {
      m[i].column = nkeys + (int)i;
      if (m[i].kind == B2_AGG_COUNT || m[i].kind == B2_AGG_COUNT_ALL) { m[i].kind = B2_AGG_SUM; m[i].out_dtype = B2_INT64; m[i].out_scale = 0; }
    }
    return m;
  }
  // a complete-mode result of one partial: the keys and the aggregates, without the counts (takes t)
  Table* without_counts(Table* t) {
    if (mode == B2_AGG_MODE_PARTIAL || counted.empty()) return t;
    TableRef in(t);
    std::vector<Column*> cols(t->cols.begin(), t->cols.begin() + keys.size() + aggs.size());
    for (Column* c : cols) col_incref(c);
    return new_table(std::move(cols));
  }
  // keys are the leading columns, then the aggregates, then the counts; keep_counts: an intermediate merge, whose result is
  // merged again, keeps the counts in every mode
  Table* merge(const Table* t, bool keep_counts = false) {
    const int nk = (int)keys.size(), na = (int)aggs.size(), nc = (int)counted.size();
    std::vector<b2_agg_spec> m = merge_specs(update_specs(), nk);
    // flag the partial decimal sums that overflowed; only when there are any does the merge carry them (MAX of the flags)
    ColsGuard flags;
    std::vector<int> flagged;
    DevBuf npois(8);
    CUDA_CHECK(cudaMemsetAsync(npois.p, 0, 8, stream()));
    for (int i = 0; i < na; i++) {
      const Column* s = t->cols[nk + i];
      if (!decimal_sum(aggs[i]) || !s->nullable() || t->rows == 0) continue;
      const int j = (int)(std::find(counted.begin(), counted.end(), i) - counted.begin());
      const int64_t* count = j < nc ? t->cols[nk + na + j]->data.as<int64_t>() : nullptr;
      Column* f = new_column(B2_INT8, 0, t->rows, false);
      flags.v.push_back(f); flagged.push_back(i);
      launch(poisoned_sums_kernel, grid_for(t->rows, 256), 256, 0, stream(), s->validity(), count, t->rows, f->data.as<int8_t>(),
             npois.as<unsigned long long>());
    }
    unsigned long long hpois = 0;
    if (!flagged.empty()) { d2h(&hpois, npois.p, 1); sync(); }
    if (hpois == 0) flagged.clear();
    std::vector<Column*> in_cols(t->cols.begin(), t->cols.end());
    for (size_t q = 0; q < flagged.size(); q++) {
      in_cols.push_back(flags.v[q]);
      m.push_back(b2_agg_spec{B2_AGG_MAX, (int)in_cols.size() - 1, B2_INT8, 0, 0});
    }
    for (Column* c : in_cols) col_incref(c);
    TableRef src(new_table(std::move(in_cols)));
    std::vector<int> cols, key_outs;   // every input column once, in order: program output i is column i
    for (int k = 0; k < nk; k++) key_outs.push_back(k);
    for (int c = 0; c < nk + (int)m.size(); c++) cols.push_back(c);
    std::unique_ptr<Program> p(make_passthrough_program(src.t, cols));
    TableRef r(scan_aggregate(p.get(), false, src.t, key_outs.data(), nk, m.data(), (int)m.size()));
    for (size_t q = 0; q < flagged.size(); q++) {
      Column* s = r.t->cols[nk + flagged[q]];
      launch(clear_poisoned_kernel, grid_for((r.t->rows + 31) / 32, 256), 256, 0, stream(), s->valid.as<uint32_t>(),
             r.t->cols[nk + na + nc + q]->data.as<int8_t>(), r.t->rows);
      s->null_count = -1;
    }
    std::vector<Column*> out(r.t->cols.begin(), r.t->cols.begin() + nk + na + (mode == B2_AGG_MODE_PARTIAL || keep_counts ? nc : 0));
    for (Column* c : out) col_incref(c);
    return new_table(std::move(out));
  }
  // first-pass aggregation of one input batch; when the device cannot hold it the batch is split in halves, each half
  // yields its own partial (the merge pass combines them like any other pair of partials)
  void first_pass(const Table* in, std::vector<TableRef>& partials, int depth) {
    try {
      const std::vector<b2_agg_spec> u = update_specs();
      partials.emplace_back(with_retry([&] { return scan_aggregate(program, has_pred, in, keys.data(), (int)keys.size(), u.data(), (int)u.size()); }));
    } catch (const Error& e) {
      if (!splittable(e) || in->rows < 2 || depth >= 12) throw;
      note_split();
      const int64_t mid = in->rows / 2;
      { TableRef lo(slice_table(in, 0, mid)); first_pass(lo.t, partials, depth + 1); }
      { TableRef hi(slice_table(in, mid, in->rows)); first_pass(hi.t, partials, depth + 1); }
    }
  }
  Table* do_next() override {
    if (rp_target > 0 && !keys.empty()) return rp_next();
    if (done) return nullptr;
    done = true;
    std::vector<TableRef> partials;
    while (true) {
      TableRef in(children[0]->next());
      if (!in.t) break;
      if (mode == B2_AGG_MODE_FINAL) partials.emplace_back(in.release());   // inputs already are aggregation buffers
      else first_pass(in.t, partials, 0);
    }
    return merge_all(partials);
  }
  Table* merge_all(std::vector<TableRef>& partials) {
    if (partials.empty()) {
      // a keyless aggregate over no batches still emits its initial-value row (GpuAggregateExec.scala:1107-1126)
      if (!keys.empty() || mode == B2_AGG_MODE_FINAL) return nullptr;
      throw Error(B2_ERR_UNSUPPORTED, "keyless aggregate over zero input batches needs the input schema");
    }
    if (partials.size() == 1 && mode != B2_AGG_MODE_FINAL) return without_counts(partials[0].release());
    std::vector<const Table*> ts;
    for (auto& p : partials) ts.push_back(p.t);
    TableRef cat(concat_tables(ts));
    return merge(cat.t);
  }

  // ---- repartitioning (GpuMergeAggregateIterator, AggregateUtils.iterateAndRepartition: GpuAggregateExec.scala:150-307, 863-1103)
  // Seeds 107 + 7 * depth, not the exchange's 42: a FINAL aggregate's input arrives split by pmod(murmur3_42(keys), world), and
  // buckets by the same hash would leave most of them empty on each rank.  Equal keys always meet in one bucket: murmur_col
  // hashes every NaN payload alike, -0.0 as 0.0 and NULL as the seed.
  static constexpr int RP_SEED = 107, RP_SEED_STEP = 7, RP_MAX_DEPTH = 10;
  int64_t rp_target = 0;   // 0: off
  int rp_parts = 16;
  int64_t rp_stats[4] = {0, 0, 0, 0};   // first-level buckets, buckets split again, bytes split, deepest level
  struct AggBucket {
    std::vector<SpillPiece> pieces;
    int64_t bytes = 0;
    int depth = 0;
  };
  std::deque<AggBucket> rp_buckets;

  // pieces are partial buffers (PARTIAL / COMPLETE) or input buffers (FINAL): the keys lead, every column is carried
  template <typename BucketOf>
  void rp_split(const Table* t, int depth, BucketOf&& bucket_of) {
    std::vector<int> kc, all;
    for (int k = 0; k < (int)keys.size(); k++) kc.push_back(k);
    for (int c = 0; c < (int)t->cols.size(); c++) all.push_back(c);
    split_pieces(t, nullptr, t->rows, kc, all, RP_SEED + RP_SEED_STEP * depth, rp_parts, [&](int p, SpillPiece&& s) {
      AggBucket& b = bucket_of(p);
      b.bytes += s.bytes;
      rp_stats[2] += s.bytes;
      b.pieces.push_back(std::move(s));
    });
  }
  // Pull phase: every piece (a first-pass partial; in FINAL mode an input batch) waits in the spill store.  When the held bytes
  // pass the target they are merged into one, counts kept; a result of at most half the target stays the only held piece, a
  // larger one is split into the first-level buckets, and so is every later piece.  True: bucketed.  False: the held pieces
  // never passed the target and are in `partials`.
  bool rp_pull(std::vector<TableRef>& partials) {
    std::vector<SpillPiece> held;
    int64_t bytes = 0;
    bool bucketed = false;
    auto first_level = [&](int p) -> AggBucket& { return rp_buckets[p]; };
    auto take = [&](TableRef piece) {
      if (bucketed) { rp_split(piece.t, 0, first_level); return; }
      held.emplace_back();
      held.back().hold(piece.t);
      bytes += held.back().bytes;
      piece.reset();
      if (bytes <= rp_target) return;
      const bool unique = held.size() == 1 && mode != B2_AGG_MODE_FINAL;   // a single partial is key-unique already
      TableRef cat(concat_pieces(held, nullptr));
      held.clear();
      TableRef merged(unique ? cat.release() : with_retry([&] { return merge(cat.t, true); }));
      cat.reset();
      if (table_bytes(merged.t) <= rp_target / 2) {
        held.emplace_back();
        held.back().hold(merged.t);
        bytes = held.back().bytes;
        return;
      }
      bucketed = true;
      rp_stats[0] = rp_parts;
      rp_buckets.resize(rp_parts);
      rp_split(merged.t, 0, first_level);
    };
    while (true) {
      TableRef in(children[0]->next());
      if (!in.t) break;
      if (mode == B2_AGG_MODE_FINAL) { take(std::move(in)); continue; }
      std::vector<TableRef> ps;
      first_pass(in.t, ps, 0);
      in.reset();
      for (auto& p : ps) take(std::move(p));
    }
    if (bucketed) return true;
    for (auto& h : held) partials.emplace_back(with_retry([&] { return h.get(); }));
    return false;
  }
  void rp_resplit() {
    AggBucket b = std::move(rp_buckets.front());
    rp_buckets.pop_front();
    const int depth = b.depth + 1;
    rp_stats[1]++;
    rp_stats[3] = std::max<int64_t>(rp_stats[3], depth);
    std::vector<AggBucket> sub(rp_parts);
    auto next_level = [&](int p) -> AggBucket& { return sub[p]; };
    for (auto& p : b.pieces) {
      TableRef t(with_retry([&] { return p.get(); }));
      p.close();
      rp_split(t.t, depth, next_level);
    }
    for (int p = rp_parts - 1; p >= 0; p--) { sub[p].depth = depth; rp_buckets.push_front(std::move(sub[p])); }
  }
  // Finish phase, one output batch per call: a bucket over the target is split again into buckets that take its place, down to
  // depth 10; otherwise adjacent buckets are taken while their bytes stay within the target (at least one) and merged
  Table* rp_next() {
    if (!done) {
      done = true;
      std::vector<TableRef> partials;
      if (!rp_pull(partials)) return merge_all(partials);
    }
    while (!rp_buckets.empty()) {
      const AggBucket& f = rp_buckets.front();
      if (f.pieces.empty()) rp_buckets.pop_front();
      else if (f.bytes > rp_target && f.depth < RP_MAX_DEPTH) rp_resplit();
      else break;
    }
    if (rp_buckets.empty()) return nullptr;
    std::vector<SpillPiece> grp;
    int64_t bytes = 0, rows = 0;
    while (!rp_buckets.empty()) {
      AggBucket& b = rp_buckets.front();
      int64_t brows = 0;
      for (auto& p : b.pieces) brows += p.rows;
      if (!grp.empty() && !b.pieces.empty() && (bytes + b.bytes > rp_target || rows + brows > 0x7fffffffLL)) break;
      bytes += b.bytes;
      rows += brows;
      for (auto& p : b.pieces) grp.push_back(std::move(p));
      rp_buckets.pop_front();
    }
    const bool unique = grp.size() == 1 && mode != B2_AGG_MODE_FINAL;   // a FINAL input batch may repeat keys
    TableRef cat(concat_pieces(grp, nullptr));
    grp.clear();
    if (unique) return without_counts(cat.release());
    return with_retry([&] { return merge(cat.t); });
  }
};

struct GpuShuffledHashJoinExec : GpuExec {  // children[0] = stream (left), children[1] = build (right)
  std::vector<int> stream_keys, build_keys;
  int kind = B2_JOIN_INNER;
  bool nulls_equal = false, built = false, full_done = false;
  // mixed join (GpuHashJoin.scala:335-530 mixed*JoinGatherMaps, :1556 ConditionalHashJoinIterator): an extra non-equi
  // condition, bound over [stream columns ++ build columns], decides which equi-matched pairs survive
  b2_handle condition = 0;
  bool pruned = false;                       // a column-pruning GpuProjectExec above the join, fused into the gathers
  std::vector<int> stream_out, build_out;    // pruned: the columns each side contributes (in this order)
  TableRef build_table;
  b2_handle ht = 0;
  // Outer joins that preserve the build side — RIGHT OUTER, and FULL OUTER with a condition — are "tracked" (HashOuterJoinIterator,
  // GpuHashJoin.scala:1807-1814): stream batches are joined one at a time (INNER / the conditional LEFT OUTER), a tracker over
  // the hash table keeps the build rows that found a partner, and once the stream side is exhausted the others come out
  // with NULL stream columns (getFinalBatch, :2288-2326).  FULL OUTER without a condition coalesces its stream side instead.
  b2_handle tracker = 0;
  TableRef stream_schema;                       // zero rows of the stream columns: the NULL side of the final rows
  Column* fin_ids = nullptr;                    // ascending ids of the unmatched build rows
  std::deque<std::pair<int64_t, int64_t>> fin;  // ranges of fin_ids still to emit
  bool fin_started = false;
  ~GpuShuffledHashJoinExec() {
    if (fin_ids) col_release(fin_ids);
    if (tracker) b2_join_tracker_close(tracker);
    if (ht) b2_join_hash_table_close(ht);
  }
  bool tracked() const { return kind == B2_JOIN_RIGHT_OUTER || (kind == B2_JOIN_FULL_OUTER && condition); }
  bool coalesced() const { return kind == B2_JOIN_FULL_OUTER && !condition; }
  void new_tracker() {   // after (re)building ht
    if (tracker) { b2_join_tracker_close(tracker); tracker = 0; }
    fin_started = false;
    if (!tracked()) return;
    int rc = b2_join_tracker_create(ht, &tracker);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
  }
  // the maps of one stream batch (through a selection vector): RIGHT OUTER probes INNER and marks the build rows it finds
  void probe(const Table* keys, Column* sel, b2_handle* lm, b2_handle* rm) {
    const b2_handle sh = sel ? to_handle(sel) : 0;
    int rc = kind == B2_JOIN_RIGHT_OUTER ? b2_join_probe_track(ht, to_handle(const_cast<Table*>(keys)), sh, B2_JOIN_INNER, tracker, lm, rm)
                                         : b2_join_probe_sel(ht, to_handle(const_cast<Table*>(keys)), sh, kind, lm, rm);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
  }
  static Table* select(const Table* t, const std::vector<int>& idx) {
    std::vector<Column*> cols;
    for (int i : idx) { if (i < 0 || i >= (int)t->cols.size()) throw Error(B2_ERR_INVALID, "join key index out of range"); col_incref(t->cols[i]); cols.push_back(t->cols[i]); }
    return new_table(std::move(cols));
  }
  void build() {
    // prepareBuildBatchesForJoin: the whole build side becomes one batch
    std::vector<TableRef> parts;
    if (sp_target > 0) {
      if (hold_build_side(parts)) { built = true; return; }
    } else {
      while (true) { TableRef b(children[1]->next()); if (!b.t) break; parts.emplace_back(b.release()); }
    }
    if (parts.empty()) throw Error(B2_ERR_UNSUPPORTED, "empty build side needs the build schema");
    if (parts.size() == 1) build_table = std::move(parts[0]);
    else { std::vector<const Table*> ts; for (auto& p : parts) ts.push_back(p.t); build_table = TableRef(concat_tables(ts)); }
    parts.clear();   // the batches are not needed once concatenated: the hash table does not wait for them to go
    TableRef bk(select(build_table.t, build_keys));
    int rc = b2_join_build(to_handle(bk.t), nulls_equal, &ht);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    new_tracker();
    built = true;
  }
  // A GpuFilterExec directly below the stream side is fused by late materialisation: the filter yields a selection vector
  // (row ids), the probe reads the keys through it and emits ORIGINAL row ids, the payload is gathered from the unfiltered
  // batch — the filtered copy of the stream side (TPC-H q3: 7.8 GB per pass over lineitem) is never written or re-read.
  GpuFilterExec* fused = nullptr;
  bool fusion_checked = false;
  int raw_col(int filter_out_col) const { return fused->keep.empty() ? filter_out_col : fused->keep[filter_out_col]; }
  // Emitting probe (join_probe_pred_emit): the maps and the payload gathers of a filtered FK -> PK join replaced by output rows
  // written from the probe kernel.  The output size is known only after the probe, and GpuCoalesceBatches above holds every
  // output batch, so columns of the batch's row count are out of the question: the first batch goes through the maps and
  // gives the matches per stream row, later batches get columns of cap = min(n, ceil(1.1 * max ratio seen * n) + 65536) rows,
  // and a batch whose matches pass cap is joined again through the maps (only the speed depends on the estimate).
  JoinPayload em_payload;
  bool em_packed = false, em_ok = false;   // payload packed (or tried); usable
  double em_ratio = -1;                    // most matches per stream row of a batch so far; < 0: no batch joined yet
  int64_t em_stats[3] = {0, 0, 0};         // batches emitted, batches joined through maps, overflow reruns
  void note_matches(int64_t matches, int64_t rows) { if (rows > 0) em_ratio = std::max(em_ratio, (double)matches / (double)rows); }
  // the output of stream batch `raw` written by the probe; nullptr: join it through the maps
  Table* try_emit(const Table* raw, int key_col, const std::vector<int>& stream_cols, int64_t* npass) {
    if (kind != B2_JOIN_INNER || tracker || em_ratio < 0 || getenv("B2_JOIN_NO_EMIT")) return nullptr;
    if (!em_packed) {
      em_packed = true;
      std::vector<int> bcols = build_out;
      if (!pruned) for (int c = 0; c < (int)build_table.t->cols.size(); c++) bcols.push_back(c);
      try { em_ok = join_pack_payload(build_table.t, bcols, em_payload); }
      catch (const Error& e) { if (e.code != B2_ERR_OOM) throw; em_ok = false; em_payload = JoinPayload(); }   // no room: the maps
    }
    if (!em_ok) return nullptr;
    const int64_t n = raw->rows;
    const int64_t cap = std::min<int64_t>(n, (int64_t)std::ceil(1.1 * em_ratio * (double)n) + 65536);
    Table* out = nullptr;
    int64_t total = 0;
    if (!join_probe_pred_emit(ht, raw, key_col, program_from(fused->program), stream_cols, em_payload, cap, &out, &total, npass)) return nullptr;
    note_matches(total, n);
    if (!out) em_stats[2]++;
    return out;
  }
  Table* fused_next() {
    TableRef raw(fused->children[0]->next());
    if (!raw.t) return nullptr;
    std::vector<int> keys, left_cols;
    for (int k : stream_keys) keys.push_back(raw_col(k));
    // simple predicate + FK -> PK inner probe: the filter is evaluated INSIDE the probe kernel (no selection vector at all)
    struct Owned { Column* c = nullptr; ~Owned() { if (c) col_release(c); } Column* take() { Column* r = c; c = nullptr; return r; } };
    Owned plm, prm, sel;
    int64_t npass = 0;
    bool in_probe = false;
    if (tracked() && !stream_schema.t) {
      std::vector<int> fcols;
      const int n = fused->keep.empty() ? (int)raw.t->cols.size() : (int)fused->keep.size();
      for (int c = 0; c < n; c++) fcols.push_back(raw_col(c));
      TableRef cols(select(raw.t, fcols));
      stream_schema = TableRef(slice_table(cols.t, 0, 0));
    }
    if (pruned) for (int c : stream_out) left_cols.push_back(raw_col(c));
    else { const int n = fused->keep.empty() ? (int)raw.t->cols.size() : (int)fused->keep.size(); for (int c = 0; c < n; c++) left_cols.push_back(raw_col(c)); }
    TableRef emitted;
    if ((kind == B2_JOIN_INNER || kind == B2_JOIN_RIGHT_OUTER) && keys.size() == 1) {
      try {
        emitted = TableRef(try_emit(raw.t, keys[0], left_cols, &npass));
        if (!emitted.t) in_probe = join_probe_pred(ht, raw.t, keys[0], program_from(fused->program), &plm.c, &prm.c, &npass, tracker);
      } catch (const Error& e) { if (!splittable(e)) throw; in_probe = false; }   // memory pressure: the selection-vector path retries and splits
    }
    auto make_sel = [&] { if (!sel.c) sel.c = run_as(fused, [&] { return filter_row_ids(program_from(fused->program), raw.t); }); };
    if (!in_probe && !emitted.t) make_sel();
    fused->num_output_rows += in_probe || emitted.t ? npass : sel.c->size; fused->num_output_batches++;
    if (emitted.t) { em_stats[0]++; return emitted.release(); }
    try {
      Table* out = with_retry([&]() -> Table* {
        Column* lmc = nullptr; Column* rmc = nullptr;
        if (plm.c) { lmc = plm.take(); rmc = prm.take(); }   // the maps of the fused kernel (first attempt only)
        else {
          make_sel();
          TableRef sk(select(raw.t, keys));
          b2_handle lm = 0, rm = 0;
          probe(sk.t, sel.c, &lm, &rm);
          lmc = col_from(lm); rmc = rm ? col_from(rm) : nullptr;
        }
        ColGuard lmap(lmc);
        ColGuard rmap(rmc);
        note_matches(lmap.c->size, raw.t->rows);
        TableRef left(gather_table(raw.t, lmap.c->data.as<int32_t>(), lmap.c->size, false, &left_cols));
        if (!rmap.c || (pruned && build_out.empty())) return left.release();
        TableRef right(gather_table(build_table.t, rmap.c->data.as<int32_t>(), rmap.c->size, kind == B2_JOIN_LEFT_OUTER, pruned ? &build_out : nullptr));
        if (pruned && stream_out.empty()) return right.release();
        std::vector<Column*> cols;
        for (auto*& c : left.t->cols) { cols.push_back(c); c = nullptr; }
        for (auto*& c : right.t->cols) { cols.push_back(c); c = nullptr; }
        left.t->cols.clear(); right.t->cols.clear();
        return new_table(std::move(cols));
      });
      em_stats[1]++;
      return out;
    } catch (const Error& e) {
      if (!splittable(e)) throw;
      // memory pressure / 2^31 limit: materialise the filter output after all and take the split-and-retry path
      std::vector<int> fcols;
      const int n = fused->keep.empty() ? (int)raw.t->cols.size() : (int)fused->keep.size();
      for (int c = 0; c < n; c++) fcols.push_back(raw_col(c));
      make_sel();
      TableRef ft(gather_table(raw.t, sel.c->data.as<int32_t>(), sel.c->size, false, &fcols));
      todo.emplace_back(std::move(ft), 0);
      return drain_todo();
    }
  }
  Table* do_next() override {
    if (!todo.empty()) return drain_todo();
    if (!fin.empty()) return final_next();
    if (!built) build();
    if (sp_active) return sp_next();
    if (!fusion_checked) {
      fusion_checked = true;
      if (kind != B2_JOIN_FULL_OUTER && !condition && !getenv("B2_NO_FILTER_FUSION")) fused = dynamic_cast<GpuFilterExec*>(children[0]);
    }
    if (fused) {
      if (Table* t = fused_next()) return t;
      return tracked() ? final_start() : nullptr;
    }
    TableRef s;
    if (coalesced()) {
      // the unmatched build rows can only be emitted once every stream row has been seen: without a condition the stream
      // side is coalesced into one batch (tracked joins keep the matched build rows across batches instead: final_start)
      if (full_done) return nullptr;
      full_done = true;
      std::vector<TableRef> parts;
      while (true) { TableRef b(children[0]->next()); if (!b.t) break; parts.emplace_back(b.release()); }
      if (parts.empty()) throw Error(B2_ERR_UNSUPPORTED, "empty stream side of a full outer join needs the stream schema");
      if (parts.size() == 1) s = std::move(parts[0]);
      else { std::vector<const Table*> ts; for (auto& q : parts) ts.push_back(q.t); s = TableRef(concat_tables(ts)); }
    } else {
      s = TableRef(children[0]->next());
    }
    if (!s.t) return tracked() ? final_start() : nullptr;
    if (tracked() && !stream_schema.t) stream_schema = TableRef(slice_table(s.t, 0, 0));
    todo.emplace_back(std::move(s), 0);
    return drain_todo();
  }
  // Tracked joins, after the last stream batch (of the pair, when sub-partitioned): the build rows never marked, NULL on the
  // stream side.  A gather that does not fit (B2_ERR_OOM after retries, B2_ERR_SIZE_OVERFLOW) is halved, so these rows may
  // come in several batches.
  Table* final_start() {
    if (fin_started) return nullptr;
    fin_started = true;
    if (!(sp_active ? sp_stream_empty.t : stream_schema.t))
      throw Error(B2_ERR_UNSUPPORTED, "empty stream side of an outer join that preserves the build side needs the stream schema");
    if (fin_ids) { col_release(fin_ids); fin_ids = nullptr; }
    fin_ids = with_retry([&] {
      b2_handle h = 0;
      int rc = b2_join_tracker_unmatched(tracker, &h);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      return col_from(h);
    });
    if (fin_ids->size) fin.emplace_back(0, fin_ids->size);
    return fin.empty() ? nullptr : final_next();
  }
  Table* final_next() {
    while (true) {
      const std::pair<int64_t, int64_t> r = fin.front();
      fin.pop_front();
      try {
        return with_retry([&] { return final_rows(r.first, r.second); });
      } catch (const Error& e) {
        if (!splittable(e) || r.second - r.first < 2) throw;
        note_split();
        const int64_t mid = r.first + (r.second - r.first) / 2;
        fin.emplace_front(mid, r.second);
        fin.emplace_front(r.first, mid);
      }
    }
  }
  Table* final_rows(int64_t lo, int64_t hi) {
    const Table* ss = sp_active ? sp_stream_empty.t : stream_schema.t;
    const int64_t n = hi - lo;
    std::vector<int> scols;
    if (pruned) scols = stream_out;
    else for (int c = 0; c < (int)ss->cols.size(); c++) scols.push_back(c);
    ColGuard oob(new_column(B2_INT32, 0, n, false));
    if (n) CUDA_CHECK(cudaMemsetAsync(oob.c->data.p, 0x80, (size_t)n * 4, stream()));   // 0x80808080 < 0: out of bounds -> NULL row
    TableRef left(gather_table(ss, oob.c->data.as<int32_t>(), n, true, &scols));
    TableRef right(gather_table(build_table.t, fin_ids->data.as<int32_t>() + lo, n, false, pruned ? &build_out : nullptr));
    return concat_cols(left.t, right.t);
  }
  // stream slices waiting to be joined (a batch that had to be split leaves its halves here; one output per next())
  std::deque<std::pair<TableRef, int>> todo;
  // one stream batch -> output batch(es).  When the gather maps would pass 2^31-1 rows (B2_ERR_SIZE_OVERFLOW) or the device
  // cannot hold the output (B2_ERR_OOM after retries) the stream batch is halved and each half joined on its own — lazily,
  // so that at most one output batch exists at a time (GpuSplitAndRetryOOM, AbstractGpuJoinIterator.scala:235-250)
  Table* drain_todo() {
    while (!todo.empty()) {
      TableRef st = std::move(todo.front().first);
      const int depth = todo.front().second;
      todo.pop_front();
      try {
        Table* out = with_retry([&] { return join_batch(st.t); });
        em_stats[1]++;
        return out;
      } catch (const Error& e) {
        if (!splittable(e) || st.t->rows < 2 || depth >= 16 || coalesced()) throw;
        note_split();
        const int64_t mid = st.t->rows / 2;
        TableRef lo, hi;
        // the halves replace the batch: the batch itself is released before they are made, so the split needs no extra room
        {
          std::vector<int> all;
          for (int c = 0; c < (int)st.t->cols.size(); c++) all.push_back(c);
          lo = TableRef(slice_table(st.t, 0, mid));
          hi = TableRef(slice_table(st.t, mid, st.t->rows));
        }
        st.reset();
        todo.emplace_front(std::move(hi), depth + 1);
        todo.emplace_front(std::move(lo), depth + 1);
      }
    }
    return nullptr;
  }
  static Table* concat_cols(Table* a, Table* b) {   // steals the columns of both
    std::vector<Column*> cols;
    for (auto*& c : a->cols) { cols.push_back(c); c = nullptr; }
    for (auto*& c : b->cols) { cols.push_back(c); c = nullptr; }
    a->cols.clear(); b->cols.clear();
    return new_table(std::move(cols));
  }
  Table* prune_pairs(const Table* pairs, int nstream) {   // [stream ++ build] -> the output columns of the node
    std::vector<Column*> cols;
    auto take = [&](int i) { col_incref(pairs->cols[i]); cols.push_back(pairs->cols[i]); };
    if (pruned) { for (int c : stream_out) take(c); for (int c : build_out) take(nstream + c); }
    else for (int i = 0; i < (int)pairs->cols.size(); i++) take(i);
    return new_table(std::move(cols));
  }
  // equi-join pairs -> condition over the pair rows -> per join type
  Table* join_batch_conditional(const Table* st) {
    TableRef sk(select(st, stream_keys));
    b2_handle lm = 0, rm = 0;
    int rc = b2_join_probe(ht, to_handle(sk.t), B2_JOIN_INNER, &lm, &rm);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    ColGuard lmap(col_from(lm)), rmap(col_from(rm));
    const int nstream = (int)st->cols.size();
    TableRef left(gather_table(st, lmap.c->data.as<int32_t>(), lmap.c->size, false, nullptr));
    TableRef right(gather_table(build_table.t, rmap.c->data.as<int32_t>(), rmap.c->size, false, nullptr));
    TableRef pairs(concat_cols(left.t, right.t));
    b2_handle ph = 0;
    rc = b2_project(condition, to_handle(pairs.t), &ph);
    if (rc != B2_OK) throw Error(rc, b2_last_error());
    TableRef pt(from_handle_owned(ph));
    Column* pass = pt.t->cols[0];
    if (pass->dtype != B2_BOOL8) throw Error(B2_ERR_INVALID, "join condition must be BOOL8");
    if (tracker) {   // the build rows of the pairs that pass (marking is idempotent: a retried or halved batch sets the same bits)
      rc = b2_join_tracker_mark(tracker, to_handle(rmap.c), to_handle(pass));
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    }
    auto stream_side = [&](const Table* t) {   // semi / anti output: the node's stream columns
      std::vector<Column*> cols;
      if (pruned) for (int c : stream_out) { col_incref(t->cols[c]); cols.push_back(t->cols[c]); }
      else for (auto* c : t->cols) { col_incref(c); cols.push_back(c); }
      return new_table(std::move(cols));
    };
    if (kind == B2_JOIN_INNER || kind == B2_JOIN_RIGHT_OUTER) {
      TableRef out(prune_pairs(pairs.t, nstream));
      return filter_by_mask(out.t, pass);
    }
    if (kind == B2_JOIN_LEFT_SEMI || kind == B2_JOIN_LEFT_ANTI) {
      ColGuard flags(rows_with_passing_pair(lmap.c, pass, st->rows, kind == B2_JOIN_LEFT_ANTI));
      TableRef side(stream_side(st));
      return filter_by_mask(side.t, flags.c);
    }
    // LEFT OUTER (and FULL OUTER's per-batch part): the passing pairs, then every stream row without one, NULL on the build side
    TableRef pruned_pairs(prune_pairs(pairs.t, nstream));
    TableRef matched(filter_by_mask(pruned_pairs.t, pass));
    ColGuard lonely(rows_with_passing_pair(lmap.c, pass, st->rows, true));
    TableRef lonely_stream(filter_by_mask(st, lonely.c));
    ColGuard oob(new_column(B2_INT32, 0, lonely_stream.t->rows, false));
    if (lonely_stream.t->rows) CUDA_CHECK(cudaMemsetAsync(oob.c->data.p, 0x80, (size_t)lonely_stream.t->rows * 4, stream()));   // 0x80808080 < 0: out of bounds -> NULL row
    TableRef nulls(gather_table(build_table.t, oob.c->data.as<int32_t>(), lonely_stream.t->rows, true, nullptr));
    TableRef lonely_pairs(concat_cols(lonely_stream.t, nulls.t));
    TableRef lonely_out(prune_pairs(lonely_pairs.t, nstream));
    // nullability must agree for the concatenation: concat_tables merges validity
    std::vector<const Table*> ts{matched.t, lonely_out.t};
    return concat_tables(ts);
  }
  Table* join_batch(const Table* st) {
    if (condition) return join_batch_conditional(st);
    TableRef sk(select(st, stream_keys));
    b2_handle lm = 0, rm = 0;
    probe(sk.t, nullptr, &lm, &rm);
    ColGuard lmap(col_from(lm));
    ColGuard rmap(rm ? col_from(rm) : nullptr);
    TableRef left(gather_table(st, lmap.c->data.as<int32_t>(), lmap.c->size, kind == B2_JOIN_FULL_OUTER, pruned ? &stream_out : nullptr));
    if (!rmap.c || (pruned && build_out.empty())) return left.release();  // semi / anti (or nothing wanted from the build side): stream columns only
    TableRef right(gather_table(build_table.t, rmap.c->data.as<int32_t>(), rmap.c->size, kind == B2_JOIN_LEFT_OUTER || kind == B2_JOIN_FULL_OUTER,
                                pruned ? &build_out : nullptr));
    if (pruned && stream_out.empty()) return right.release();
    std::vector<Column*> cols;  // output = left columns ++ right columns (GpuHashJoin.scala:2451-2470)
    for (auto*& c : left.t->cols) { cols.push_back(c); c = nullptr; }
    for (auto*& c : right.t->cols) { cols.push_back(c); c = nullptr; }
    left.t->cols.clear(); right.t->cols.clear();
    return new_table(std::move(cols));
  }

  // ---- GpuSubPartitionHashJoin (GpuSubPartitionHashJoin.scala) -------------------------------------------------------------
  // Seeds 100 and 110, not the exchange's 42: rows reach this node already assigned by pmod(murmur3_42, world), and buckets by
  // the same hash would leave only K / gcd(K, world) of the K buckets non-empty on each rank.
  static constexpr int SP_SEED = 100, SP_RESEED = 110;
  int64_t sp_target = 0;   // 0: off
  int sp_parts = 16;
  int64_t sp_stats[4] = {0, 0, 0, 0};
  bool sp_active = false, sp_read = false;
  struct Bucket {
    std::vector<SpillPiece> build, stream;
    int64_t build_bytes = 0, stream_bytes = 0;
    bool resplit = false;   // made by repartitioning a bucket: never split again
  };
  std::deque<Bucket> sp_buckets;
  std::deque<std::vector<SpillPiece>> sp_probe;   // the open pair's stream pieces, one group per probe batch
  TableRef sp_build_empty, sp_stream_empty;       // zero-row tables of the carried columns
  std::vector<int> sp_bkeys, sp_bkeep;            // first-level split of the build batches: keys and carried columns

  // the columns one side carries through its buckets: with pruning and no condition the keys and the output columns (indices
  // remapped), otherwise every column
  std::vector<int> carried(int ncols, std::vector<int>& keys, std::vector<int>& out_cols) {
    std::vector<int> keep;
    if (!pruned || condition) { for (int c = 0; c < ncols; c++) keep.push_back(c); return keep; }
    auto pos = [&](int c) {
      if (c < 0 || c >= ncols) throw Error(B2_ERR_INVALID, "join column index out of range");
      for (size_t k = 0; k < keep.size(); k++) if (keep[k] == c) return (int)k;
      keep.push_back(c);
      return (int)keep.size() - 1;
    };
    for (int& k : keys) k = pos(k);
    for (int& c : out_cols) c = pos(c);
    return keep;
  }
  template <typename BucketOf>
  void split_into(const Table* t, const int32_t* d_sel, int64_t n, const std::vector<int>& keys, const std::vector<int>& keep, int seed, int nparts,
                  BucketOf&& bucket_of, bool build_side, int64_t* bytes_out) {
    split_pieces(t, d_sel, n, keys, keep, seed, nparts, [&](int p, SpillPiece&& s) {
      Bucket& b = bucket_of(p);
      (build_side ? b.build_bytes : b.stream_bytes) += s.bytes;
      if (bytes_out) *bytes_out += s.bytes;
      (build_side ? b.build : b.stream).push_back(std::move(s));
    });
  }
  // Pulls the build side into the spill store.  False: it stayed within the target and `parts` holds its batches.  True: it
  // passed the target and is split into the buckets.
  bool hold_build_side(std::vector<TableRef>& parts) {
    std::vector<SpillPiece> held;
    int64_t bytes = 0;
    auto first_level = [&](int p) -> Bucket& { return sp_buckets[p]; };
    auto split = [&](const Table* t) { split_into(t, nullptr, t->rows, sp_bkeys, sp_bkeep, SP_SEED, sp_parts, first_level, true, &sp_stats[2]); };
    while (true) {
      TableRef b(children[1]->next());
      if (!b.t) break;
      if (sp_active) { split(b.t); continue; }
      bytes += table_bytes(b.t);
      held.emplace_back();
      held.back().hold(b.t);
      if (bytes <= sp_target) continue;
      sp_active = true;
      sp_stats[0] = sp_parts;
      sp_buckets.resize(sp_parts);
      sp_bkeys = build_keys;
      sp_bkeep = carried((int)b.t->cols.size(), build_keys, build_out);
      { TableRef sel(select(b.t, sp_bkeep)); sp_build_empty = TableRef(slice_table(sel.t, 0, 0)); }
      b.reset();
      for (auto& h : held) {
        TableRef t(with_retry([&] { return h.get(); }));
        h.close();
        split(t.t);
      }
      held.clear();
    }
    if (sp_active) return true;
    for (auto& h : held) parts.emplace_back(with_retry([&] { return h.get(); }));
    return false;
  }
  // The stream side, split by the same keys, seed and K; through the selection vector of a GpuFilterExec directly below
  void split_stream_side() {
    GpuFilterExec* ff = nullptr;
    if (kind != B2_JOIN_FULL_OUTER && !condition && !getenv("B2_NO_FILTER_FUSION")) ff = dynamic_cast<GpuFilterExec*>(children[0]);
    std::vector<int> keys, keep;   // indices into the batches pulled (the filter's input when fused)
    auto first_level = [&](int p) -> Bucket& { return sp_buckets[p]; };
    while (true) {
      TableRef raw(ff ? ff->children[0]->next() : children[0]->next());
      if (!raw.t) break;
      if (keep.empty()) {
        const int ncols = ff && !ff->keep.empty() ? (int)ff->keep.size() : (int)raw.t->cols.size();
        auto raw_of = [&](int c) { return ff && !ff->keep.empty() ? ff->keep[c] : c; };
        for (int k : stream_keys) keys.push_back(raw_of(k));
        for (int c : carried(ncols, stream_keys, stream_out)) keep.push_back(raw_of(c));
        TableRef sel(select(raw.t, keep));
        sp_stream_empty = TableRef(slice_table(sel.t, 0, 0));
      }
      ColGuard sel(ff ? run_as(ff, [&] { return filter_row_ids(program_from(ff->program), raw.t); }) : nullptr);
      if (ff) { ff->num_output_rows += sel.c->size; ff->num_output_batches++; }
      split_into(raw.t, sel.c ? sel.c->data.as<int32_t>() : nullptr, sel.c ? sel.c->size : raw.t->rows, keys, keep, SP_SEED, sp_parts,
                 first_level, false, &sp_stats[3]);
    }
    if (!sp_stream_empty.t && (coalesced() || tracked()))
      throw Error(B2_ERR_UNSUPPORTED, "empty stream side of an outer join that preserves the build side needs the stream schema");
  }
  bool useless(const Bucket& b) const {
    if (kind == B2_JOIN_INNER || kind == B2_JOIN_LEFT_SEMI) return b.build.empty() || b.stream.empty();
    if (kind == B2_JOIN_FULL_OUTER) return b.build.empty() && b.stream.empty();
    if (kind == B2_JOIN_RIGHT_OUTER) return b.build.empty();   // build rows without stream rows are still output
    return b.stream.empty();   // LEFT OUTER / ANTI: stream rows without build rows are still output
  }
  // GpuSubPartitionPairIterator: a bucket still over the target is split once more, with its stream pieces.  FULL OUTER without
  // a condition coalesces a pair's stream side, so there a bucket whose stream pieces pass the target is split again as well.
  void repartition() {
    Bucket b = std::move(sp_buckets.front());
    sp_buckets.pop_front();
    sp_stats[1]++;
    const int64_t bytes = std::max(b.build_bytes, coalesced() ? b.stream_bytes : 0);
    const int k2 = (int)std::min<int64_t>(256, std::max<int64_t>(sp_parts, bytes / sp_target + 1));
    std::vector<Bucket> sub(k2);
    auto second_level = [&](int p) -> Bucket& { return sub[p]; };
    std::vector<int> all_b, all_s;
    for (int c = 0; c < (int)sp_build_empty.t->cols.size(); c++) all_b.push_back(c);
    for (int c = 0; sp_stream_empty.t && c < (int)sp_stream_empty.t->cols.size(); c++) all_s.push_back(c);
    for (auto& p : b.build) { TableRef t(with_retry([&] { return p.get(); })); p.close(); split_into(t.t, nullptr, t.t->rows, build_keys, all_b, SP_RESEED, k2, second_level, true, nullptr); }
    for (auto& p : b.stream) { TableRef t(with_retry([&] { return p.get(); })); p.close(); split_into(t.t, nullptr, t.t->rows, stream_keys, all_s, SP_RESEED, k2, second_level, false, nullptr); }
    for (int p = k2 - 1; p >= 0; p--) { sub[p].resplit = true; sp_buckets.push_front(std::move(sub[p])); }
  }
  // GpuBatchSubPartitionIterator: the next pair = adjacent useful buckets whose build pieces together stay within the target.
  // Builds its hash table (and tracker) and queues its stream pieces in probe groups of at most the target (FULL OUTER without a
  // condition: one group).
  bool open_next_pair() {
    if (tracker) { b2_join_tracker_close(tracker); tracker = 0; }
    if (ht) { b2_join_hash_table_close(ht); ht = 0; }
    build_table.reset();
    auto over = [&](const Bucket& b) {
      return !b.resplit && (b.build_bytes > sp_target || (coalesced() && b.stream_bytes > sp_target));
    };
    while (!sp_buckets.empty()) {
      if (useless(sp_buckets.front())) sp_buckets.pop_front();
      else if (over(sp_buckets.front())) repartition();
      else break;
    }
    if (sp_buckets.empty()) return false;
    // FULL OUTER without a condition coalesces the pair's stream side as well, so its stream pieces count against the target too
    const bool full = coalesced();
    std::vector<Bucket> pair;
    int64_t bytes = sp_buckets.front().build_bytes, sbytes = sp_buckets.front().stream_bytes;
    pair.push_back(std::move(sp_buckets.front()));
    sp_buckets.pop_front();
    while (!sp_buckets.empty()) {
      const Bucket& nb = sp_buckets.front();
      if (useless(nb)) { sp_buckets.pop_front(); continue; }
      if (over(nb) || bytes + nb.build_bytes > sp_target || (full && sbytes + nb.stream_bytes > sp_target)) break;
      bytes += nb.build_bytes; sbytes += nb.stream_bytes;
      pair.push_back(std::move(sp_buckets.front()));
      sp_buckets.pop_front();
    }
    std::vector<SpillPiece> bp, sps;
    for (auto& b : pair) {
      for (auto& p : b.build) bp.push_back(std::move(p));
      for (auto& p : b.stream) sps.push_back(std::move(p));
    }
    build_table = TableRef(concat_pieces(bp, sp_build_empty.t));
    bp.clear();
    ht = with_retry([&] {
      TableRef bk(select(build_table.t, build_keys));
      b2_handle h = 0;
      int rc = b2_join_build(to_handle(bk.t), nulls_equal, &h);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      return h;
    });
    new_tracker();
    if (full) { sp_probe.push_back(std::move(sps)); return true; }
    std::vector<SpillPiece> grp;
    int64_t gb = 0, gr = 0;
    for (auto& p : sps) {
      if (!grp.empty() && (gb + p.bytes > sp_target || gr + p.rows > 0x7fffffffLL)) { sp_probe.push_back(std::move(grp)); grp.clear(); gb = gr = 0; }
      gb += p.bytes; gr += p.rows;
      grp.push_back(std::move(p));
    }
    if (!grp.empty()) sp_probe.push_back(std::move(grp));
    return true;
  }
  Table* sp_next() {
    if (!sp_read) { sp_read = true; split_stream_side(); }
    while (true) {
      if (!todo.empty()) return drain_todo();
      if (!fin.empty()) return final_next();
      if (!sp_probe.empty()) {
        std::vector<SpillPiece> grp = std::move(sp_probe.front());
        sp_probe.pop_front();
        todo.emplace_back(TableRef(concat_pieces(grp, sp_stream_empty.t)), 0);
        continue;
      }
      if (ht && tracked() && !fin_started) {   // the pair's last group is done (or it had none): its unmatched build rows
        if (Table* t = final_start()) return t;
        continue;
      }
      if (!open_next_pair()) return nullptr;
    }
  }
};

DevBuf sort_order(const Table* t, const b2_order_by_arg* keys, int nkeys);
Table* top_n_table(const Table* t, const b2_order_by_arg* keys, int nkeys, int64_t limit);
struct GpuSortExec : GpuExec {
  std::vector<b2_order_by_arg> order;
  bool global = true;   // false: sort each batch (SortEachBatch); true: full sort of the partition
  int64_t limit = -1;   // >= 0: GpuTopN
  bool done = false;
  Table* sorted(const Table* t, int64_t n) {
    if (n >= 0) return top_n_table(t, order.data(), (int)order.size(), n);   // GpuTopN: radix select, then a sort of the candidates
    DevBuf perm = sort_order(t, order.data(), (int)order.size());
    return gather_table(t, perm.as<int32_t>(), n < 0 ? t->rows : std::min<int64_t>(n, t->rows), false, nullptr);
  }
  Table* do_next() override {
    if (!global && limit < 0) {
      TableRef in(children[0]->next());
      return in.t ? sorted(in.t, -1) : nullptr;
    }
    if (done) return nullptr;
    done = true;
    TableRef pending;
    std::vector<TableRef> all;   // full sort: every batch, concatenated once
    while (true) {
      TableRef in(children[0]->next());
      if (!in.t) break;
      if (limit >= 0) {
        // GpuTopN: sort the batch, keep N, fold into the running top-N
        TableRef top(sorted(in.t, limit));
        if (!pending.t) pending = std::move(top);
        else { std::vector<const Table*> ts{pending.t, top.t}; TableRef cat(concat_tables(ts)); pending = TableRef(sorted(cat.t, limit)); }
      } else {
        all.push_back(std::move(in));
      }
    }
    if (limit >= 0) return pending.release();
    if (all.empty()) return nullptr;
    if (all.size() == 1) return sorted(all[0].t, -1);
    std::vector<const Table*> ts;
    for (auto& a : all) ts.push_back(a.t);
    TableRef cat(concat_tables(ts));
    all.clear();
    return sorted(cat.t, -1);
  }
};

DevBuf merge_runs(const Table* t, const std::vector<int64_t>& off, const b2_order_by_arg* keys, int nkeys, const int64_t* tie);   // sort.cu
int64_t lower_bound_row(const Table* sorted, const Table* probe, const b2_order_by_arg* keys, int nkeys);

__global__ void ordinal_kernel(int64_t* __restrict__ out, int64_t n, int64_t base) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = base + i;
}

// GpuOutOfCoreSortIterator (GpuSortExec.scala:241-630): a full sort of a partition that need not fit on the device.
//  1. Every input batch gets an INT64 ordinal column (input position: batch base + row), is sorted (stable, so the ordinal needs
//     no radix digits) and cut into spillable pieces of at most target/8 bytes.  With the ordinal as the last key the order is
//     strict: "row x comes before row y" has one answer, which makes the cut below exact and the whole sort stable.
//  2. A round takes the pending pieces with the smallest first rows (ordered by a device sort of a table of those rows) until
//     the window would pass the target, merges them (merge_runs), and keeps as final every merged row that sorts before the
//     first row of the smallest piece left pending (lower_bound_row).  The rest is cut into pieces again.  The window holds the
//     smallest pending piece and its first row sorts before every other first row, so each round finalises at least one row.
//  3. Final pieces are concatenated up to the target, and the ordinal is dropped.
// Every device step runs under with_retry: an OOM spills the idle pieces to the host and tries again.  Output batches are at
// most `target` bytes as the spill store counts them (table_bytes), unless a single row is larger, and below 2^31 rows.
struct GpuOutOfCoreSortExec : GpuExec {
  std::vector<b2_order_by_arg> order;        // the sort keys
  std::vector<b2_order_by_arg> merge_keys;   // the sort keys, then the ordinal
  int64_t target = 0;
  struct Piece : SpillPiece {
    // pending pieces: their first row, kept on the device outside the spill store (one row per piece, and there are at most
    // about 8 pieces per target_bytes of input) so that ordering the pieces never brings a spilled piece back
    TableRef head;
    Piece() {}
    Piece(Piece&&) noexcept = default;
    Piece& operator=(Piece&&) noexcept = default;
  };
  std::vector<Piece> pending;
  std::deque<Piece> final_q;
  int64_t final_bytes = 0, ordinal_base = 0;
  std::vector<int> dtypes;
  bool read = false;

  // rows [from, to) of the sorted table `t`, cut into pieces of at most `limit` bytes (a single row may be larger)
  std::vector<Piece> cut(const Table* t, int64_t from, int64_t to, int64_t limit, bool with_heads) {
    const int nc = (int)t->cols.size();
    std::vector<std::vector<int32_t>> offs(nc);   // host copies of the string offsets: piece sizes are exact
    for (int c = 0; c < nc; c++)
      if (t->cols[c]->dtype == B2_STRING && to > from) {
        offs[c].resize((size_t)(to - from + 1));
        d2h(offs[c].data(), t->cols[c]->offsets.as<int32_t>() + from, offs[c].size());
      }
    sync();
    auto bytes = [&](int64_t s, int64_t e) {
      const int64_t n = e - s;
      int64_t b = 0;
      for (int c = 0; c < nc; c++) {
        const Column* col = t->cols[c];
        if (col->dtype == B2_STRING) b += (int64_t)offs[c][e - from] - offs[c][s - from] + (n + 1) * 4;
        else b += n * dtype_width(col->dtype);
        if (col->nullable()) b += (int64_t)validity_bytes(n);
      }
      return b;
    };
    std::vector<Piece> out;
    for (int64_t s = from; s < to;) {
      int64_t lo = s + 1, hi = to;   // the largest e in [s+1, to] with bytes(s, e) <= limit, at least s+1
      while (lo < hi) { const int64_t mid = lo + (hi - lo + 1) / 2; if (bytes(s, mid) <= limit) lo = mid; else hi = mid - 1; }
      const int64_t e = lo;
      TableRef piece(slice_table(t, s, e));
      Piece p;
      if (with_heads) p.head = TableRef(slice_table(t, s, s + 1));
      p.hold(piece.t);
      out.push_back(std::move(p));
      s = e;
    }
    return out;
  }

  // table_bytes of the concatenation of `n` final pieces without the ordinal
  int64_t output_bytes(size_t n) const {
    int64_t rows = 0;
    for (size_t i = 0; i < n; i++) rows += final_q[i].rows;
    int64_t b = 0;
    for (size_t c = 0; c + 1 < dtypes.size(); c++) {
      bool nullable = false;
      for (size_t i = 0; i < n; i++) { nullable = nullable || final_q[i].nullable[c]; if (dtypes[c] == B2_STRING) b += final_q[i].chars[c]; }
      b += dtypes[c] == B2_STRING ? (rows + 1) * 4 : rows * dtype_width(dtypes[c]);
      if (nullable) b += (int64_t)validity_bytes(rows);
    }
    return b;
  }

  void first_pass() {
    while (true) {
      TableRef in(children[0]->next());
      if (!in.t) break;
      if (in.t->rows == 0) continue;
      if (dtypes.empty()) {
        for (const auto& k : order)   // before the ordinal is appended, which a key one past the last column would name
          B2_CHECK(k.column >= 0 && k.column < (int)in.t->cols.size(), "sort key column out of range");
        for (const Column* c : in.t->cols) dtypes.push_back(c->dtype);
        dtypes.push_back(B2_INT64);
        merge_keys = order;
        merge_keys.push_back(b2_order_by_arg{(int32_t)in.t->cols.size(), 1, 1});
      }
      std::vector<Piece> pieces = with_retry([&] {
        ColGuard ord(new_column(B2_INT64, 0, in.t->rows, false));
        launch(ordinal_kernel, grid_for(in.t->rows, 256), 256, 0, stream(), ord.c->data.as<int64_t>(), in.t->rows, ordinal_base);
        std::vector<Column*> cols(in.t->cols.begin(), in.t->cols.end());
        for (Column* c : cols) col_incref(c);
        cols.push_back(ord.release());
        TableRef with_ord(new_table(std::move(cols)));
        DevBuf perm = sort_order(with_ord.t, order.data(), (int)order.size());
        TableRef sorted(gather_table(with_ord.t, perm.as<int32_t>(), with_ord.t->rows, false, nullptr));
        with_ord.reset();
        perm.reset();
        return cut(sorted.t, 0, sorted.t->rows, target / 8, true);
      });
      ordinal_base += in.t->rows;
      for (auto& p : pieces) pending.push_back(std::move(p));
    }
  }

  void merge_round() {
    if (pending.size() > 1) {   // order the pending pieces by their first rows, on the device
      std::vector<int32_t> rank = with_retry([&] {
        std::vector<const Table*> hs;
        for (auto& p : pending) hs.push_back(p.head.t);
        TableRef heads(concat_tables(hs));
        DevBuf perm = sort_order(heads.t, merge_keys.data(), (int)merge_keys.size());
        std::vector<int32_t> h(pending.size());
        d2h(h.data(), perm.p, h.size());
        sync();
        return h;
      });
      std::vector<Piece> by_head;
      for (int32_t r : rank) by_head.push_back(std::move(pending[r]));
      pending.swap(by_head);
    }
    size_t take = 0;
    int64_t bytes = 0, rows = 0;
    while (take < pending.size() && (take == 0 || (bytes + pending[take].bytes <= target && rows + pending[take].rows <= 0x7fffffffLL))) {
      bytes += pending[take].bytes; rows += pending[take].rows; take++;
    }
    if (take == pending.size() && take == 1) {   // the last pending piece: final as it stands
      final_bytes += pending[0].bytes;
      pending[0].head.reset();
      final_q.push_back(std::move(pending[0]));
      pending.clear();
      return;
    }
    std::pair<std::vector<Piece>, std::vector<Piece>> cuts = with_retry([&] {
      TableRef merged;
      {
        std::vector<TableRef> win;
        std::vector<const Table*> ts;
        std::vector<int64_t> off{0};
        for (size_t i = 0; i < take; i++) { win.emplace_back(pending[i].get()); ts.push_back(win.back().t); off.push_back(off.back() + win.back().t->rows); }
        TableRef cat(concat_tables(ts));
        win.clear();   // the pieces stay in the spill store (and may leave the device) until the round has succeeded
        // the ordinal is the tie-break: compared as a plain INT64, not through the normalised key
        DevBuf perm = merge_runs(cat.t, off, order.data(), (int)order.size(), cat.t->cols.back()->data.as<int64_t>());
        merged = TableRef(gather_table(cat.t, perm.as<int32_t>(), cat.t->rows, false, nullptr));
      }
      const int64_t n = merged.t->rows;
      const int64_t fin = take == pending.size() ? n : lower_bound_row(merged.t, pending[take].head.t, merge_keys.data(), (int)merge_keys.size());
      if (fin < 1) throw Error(B2_ERR_INVALID, "out-of-core sort: a merge round finalised no row");
      return std::make_pair(cut(merged.t, 0, fin, target / 8, false), cut(merged.t, fin, n, target / 8, true));
    });
    for (auto& p : cuts.first) { final_bytes += p.bytes; final_q.push_back(std::move(p)); }
    pending.erase(pending.begin(), pending.begin() + take);
    for (auto& p : cuts.second) pending.push_back(std::move(p));
  }

  Table* do_next() override {
    if (!read) { read = true; first_pass(); }
    while (!pending.empty() && final_bytes < target) merge_round();
    if (final_q.empty()) return nullptr;
    size_t n = 1;
    int64_t rows = final_q[0].rows;
    while (n < final_q.size() && rows + final_q[n].rows <= 0x7fffffffLL && output_bytes(n + 1) <= target) rows += final_q[n++].rows;
    Table* out = with_retry([&] {
      std::vector<TableRef> parts;
      for (size_t i = 0; i < n; i++) {
        TableRef t(final_q[i].get());
        std::vector<Column*> cols(t.t->cols.begin(), t.t->cols.end() - 1);   // without the ordinal
        for (Column* c : cols) col_incref(c);
        parts.emplace_back(new_table(std::move(cols)));
      }
      if (n == 1) return parts[0].release();
      std::vector<const Table*> ts;
      for (auto& p : parts) ts.push_back(p.t);
      return concat_tables(ts);
    });
    for (size_t i = 0; i < n; i++) { final_bytes -= final_q.front().bytes; final_q.pop_front(); }
    return out;
  }
};

struct GpuCoalesceBatches : GpuExec {
  int64_t target_rows = 1 << 30;
  TableRef carry;
  Table* do_next() override {
    std::vector<TableRef> acc;
    int64_t rows = 0;
    if (carry.t) { rows += carry.t->rows; acc.emplace_back(carry.release()); }
    while (rows < target_rows) {
      TableRef in(children[0]->next());
      if (!in.t) break;
      if (rows > 0 && rows + in.t->rows > target_rows) { carry = std::move(in); break; }
      rows += in.t->rows;
      acc.emplace_back(in.release());
    }
    if (acc.empty()) return nullptr;
    if (acc.size() == 1) return acc[0].release();
    std::vector<const Table*> ts;
    for (auto& a : acc) ts.push_back(a.t);
    return concat_tables(ts);
  }
};

extern "C" int b2_exchange_hash(b2_handle comm, b2_handle table, const int32_t* key_cols, int32_t nkeys, int32_t seed, b2_handle* out_table, int32_t* any_data);
extern "C" int b2_exchange_ex(b2_handle comm, b2_handle partitioned_table, const int32_t* offsets, b2_handle* out_table, int32_t* any_data);
extern "C" int b2_comm_fused_ready(b2_handle comm, int32_t* ok);
extern "C" int b2_comm_allmax(b2_handle comm, int32_t value, int32_t* out);
extern "C" int b2_exchange_hash_sel(b2_handle comm, b2_handle table, b2_handle selection, const int32_t* out_cols, int32_t nout, const int32_t* key_cols,
                                    int32_t nkeys, int32_t seed, b2_handle* out_table, int32_t* any_data);
extern "C" int b2_broadcast_table(b2_handle comm, b2_handle table, int32_t root, b2_handle* out_table);

// GpuShuffleExchangeExec (GpuShuffleExchangeExecBase.scala:384-536).  Every call of the exchange is a collective, so the
// node follows a termination protocol instead of stopping when ITS child is exhausted: a rank without a batch keeps
// taking part (sending nothing) until no rank has data left — ranks with different batch counts, or with none at all,
// cannot strand their peers (the reference's pull-based shuffle has no such constraint).
struct GpuShuffleExchangeExec : GpuExec {
  std::vector<int32_t> key_cols;   // empty = SinglePartition (everything to rank 0)
  b2_handle comm = 0;
  int world = 1;
  bool finished = false, probed = false, fused = false;
  Table* do_next() override {
    if (finished) return nullptr;
    if (world == 1 || !comm) {
      TableRef in(children[0]->next());
      if (!in.t) { finished = true; return nullptr; }
      if (key_cols.empty()) return in.release();
      std::vector<int32_t> offs(world + 1, 0);
      b2_handle out = 0;
      int rc = b2_hash_partition(to_handle(in.t), key_cols.data(), (int)key_cols.size(), 42, world, &out, offs.data());
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      return from_handle_owned(out);
    }
    // a GpuFilterExec (with its column pruning) directly below is fused into the scatter: see GpuShuffledHashJoinExec::fused
    GpuFilterExec* ff = getenv("B2_NO_FILTER_FUSION") ? nullptr : dynamic_cast<GpuFilterExec*>(children[0]);
    GpuExec* src = ff ? ff->children[0] : children[0];
    // one batch of look-ahead: the call that carries a rank's LAST batch says so (b2_comm_set_more), and when no rank has
    // more the exchange is over without an extra, empty round (one header all-gather + D2H + sync per exchange node)
    if (!primed) { primed = true; ahead = TableRef(src->next()); }
    TableRef in = std::move(ahead);
    if (in.t) ahead = TableRef(src->next());
    {
      int rc = b2_comm_set_more(comm, ahead.t ? 1 : 0);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    }
    std::vector<int32_t> out_cols;     // the columns that travel (indices into the batch pulled from src)
    if (ff && in.t) {
      if (ff->keep.empty()) for (int c = 0; c < (int)in.t->cols.size(); c++) out_cols.push_back(c);
      else out_cols = ff->keep;
    }
    if (!probed) {   // collective, once per node: can every rank store into every peer's arena, and is the schema fixed width?
      int32_t ok = 0;
      int rc = b2_comm_fused_ready(comm, &ok);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      // a rank without a batch does not know the schema, so the ranks agree on "some batch carries STRING columns"
      int32_t mine = 0, any_strings = 0;
      if (in.t && !ff) for (auto* c : in.t->cols) if (c->dtype == B2_STRING) mine = 1;
      if (in.t && ff) for (int c : out_cols) if (in.t->cols[c]->dtype == B2_STRING) mine = 1;
      rc = b2_comm_allmax(comm, mine, &any_strings);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      has_strings = any_strings != 0;
      fused = ok != 0; probed = true;
    }
    b2_handle out = 0;
    int32_t any = 0;
    if (fused && !has_strings && ff) {
      ColGuard sel(in.t ? run_as(ff, [&] { return filter_row_ids(program_from(ff->program), in.t); }) : nullptr);
      if (in.t) { ff->num_output_rows += sel.c->size; ff->num_output_batches++; }
      std::vector<int32_t> keys;   // key_cols index the filter's output columns
      for (int32_t k : key_cols) keys.push_back(ff->keep.empty() ? k : ff->keep[k]);
      int rc = b2_exchange_hash_sel(comm, in.t ? to_handle(in.t) : 0, sel.c ? to_handle(sel.c) : 0, out_cols.data(), (int)out_cols.size(), keys.data(),
                                    (int)keys.size(), 42, &out, &any);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    } else if (fused && !has_strings) {
      int rc = b2_exchange_hash(comm, in.t ? to_handle(in.t) : 0, key_cols.data(), (int)key_cols.size(), 42, &out, &any);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    } else {
      if (ff && in.t) {   // NCCL path: the filter runs unfused
        TableRef f(ff->keep.empty() ? nullptr : filter_select(program_from(ff->program), in.t, ff->keep.data(), (int)ff->keep.size()));
        if (!f.t) { b2_handle fh = 0; int rc = b2_filter(ff->program, to_handle(in.t), &fh); if (rc != B2_OK) throw Error(rc, b2_last_error()); f = TableRef(from_handle_owned(fh)); }
        ff->num_output_rows += f.t->rows; ff->num_output_batches++;
        in = std::move(f);
      }
      std::vector<int32_t> offs(world + 1, 0);
      TableRef part;
      if (in.t) {
        if (key_cols.empty()) {
          in.t->refs.fetch_add(1);
          part = TableRef(in.t);
          for (int r = 1; r <= world; r++) offs[r] = (int32_t)in.t->rows;
        } else {
          b2_handle ph = 0;
          int rc = b2_hash_partition(to_handle(in.t), key_cols.data(), (int)key_cols.size(), 42, world, &ph, offs.data());
          if (rc != B2_OK) throw Error(rc, b2_last_error());
          part = TableRef(from_handle_owned(ph));
        }
      }
      int rc = b2_exchange_ex(comm, part.t ? to_handle(part.t) : 0, part.t ? offs.data() : nullptr, &out, &any);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    }
    int32_t any_more = 1;
    {
      int rc = b2_comm_any_more(comm, &any_more);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
    }
    if (!any_more) finished = true;            // every rank sent its last batch (or had none): no further round
    if (!any) { finished = true; if (out) table_release(from_handle_owned(out)); return nullptr; }
    return from_handle_owned(out);
  }
  bool primed = false;
  TableRef ahead;             // the batch the NEXT call will carry
  bool has_strings = false;   // the path (fused / NCCL) is a per-node property every rank agrees on at the first call
};

// GpuBroadcastExchangeExec (GpuBroadcastExchangeExec.scala:1-664): the child relation is collected once and every rank gets
// the WHOLE relation.  SPMD form: each rank coalesces its slice and broadcasts it (ncclBroadcast per rank), the result is
// the concatenation in rank order.  One batch out.
struct GpuBroadcastExchangeExec : GpuExec {
  b2_handle comm = 0;
  int world = 1, rank = 0;
  bool done = false;
  std::vector<int> schema_dtype, schema_scale;   // needed when this rank's slice is empty
  Table* do_next() override {
    if (done) return nullptr;
    done = true;
    std::vector<TableRef> parts;
    while (true) { TableRef b(children[0]->next()); if (!b.t) break; parts.emplace_back(b.release()); }
    TableRef mine;
    if (parts.size() == 1) mine = std::move(parts[0]);
    else if (parts.size() > 1) { std::vector<const Table*> ts; for (auto& p : parts) ts.push_back(p.t); mine = TableRef(concat_tables(ts)); }
    if (world == 1 || !comm) return mine.release();
    if (!mine.t) throw Error(B2_ERR_UNSUPPORTED, "broadcast of a slice with no batches needs the schema (push an empty batch)");
    std::vector<TableRef> got;
    for (int r = 0; r < world; r++) {
      b2_handle out = 0;
      int rc = b2_broadcast_table(comm, r == rank ? to_handle(mine.t) : 0, r, &out);
      if (rc != B2_OK) throw Error(rc, b2_last_error());
      got.emplace_back(from_handle_owned(out));
    }
    std::vector<const Table*> ts;
    for (auto& g : got) ts.push_back(g.t);
    return concat_tables(ts);
  }
};

}  // namespace b2

using namespace b2;
extern "C" {

int b2_exec_source(b2_handle* out) {
  B2_TRY
  *out = to_handle(new GpuBatchSource());
  B2_CATCH
}
int b2_exec_source_push(b2_handle src, b2_handle table) {
  B2_TRY
  auto* s = dynamic_cast<GpuBatchSource*>(exec_from(src));
  B2_CHECK(s, "not a batch source");
  Table* t = table_from(table);
  t->refs.fetch_add(1);
  s->q.push_back(t);
  B2_CATCH
}
int b2_exec_parquet_scan(const char* const* column_names, int32_t ncols, b2_handle* out) {
  B2_TRY
  auto* e = new GpuParquetScanExec();
  for (int i = 0; i < ncols; i++) e->names.push_back(column_names[i]);
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_parquet_scan_add(b2_handle scan, const uint8_t* host_buf, int64_t len) {
  B2_TRY
  auto* s = dynamic_cast<GpuParquetScanExec*>(exec_from(scan));
  B2_CHECK(s, "not a parquet scan");
  s->bufs.push_back({host_buf, len});
  B2_CATCH
}
int b2_exec_filter(b2_handle child, b2_handle predicate_program, b2_handle* out) {
  B2_TRY
  auto* e = new GpuFilterExec();
  e->add_child(exec_from(child)); e->program = predicate_program;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_filter_select(b2_handle child, b2_handle predicate_program, const int32_t* keep_cols, int32_t nkeep, b2_handle* out) {
  B2_TRY
  B2_CHECK(nkeep >= 1, "filter: at least one output column");
  auto* e = new GpuFilterExec();
  e->add_child(exec_from(child)); e->program = predicate_program;
  e->keep.assign(keep_cols, keep_cols + nkeep);
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_host_source(b2_handle* out) {
  B2_TRY
  *out = to_handle(new GpuHostBatchSource());
  B2_CATCH
}
int b2_exec_host_source_push(b2_handle source, const b2_host_column* cols, int32_t ncols) {
  B2_TRY
  auto* s = dynamic_cast<GpuHostBatchSource*>(exec_from(source));
  B2_CHECK(s, "not a host batch source");
  B2_CHECK(ncols >= 1, "a batch needs columns");
  std::vector<HostColumn> b;
  for (int i = 0; i < ncols; i++) {
    B2_CHECK(cols[i].rows == cols[0].rows, "host batch columns differ in length");
    b.push_back({cols[i].dtype, cols[i].scale, cols[i].rows, cols[i].data, cols[i].validity_bits, cols[i].offsets});
  }
  s->batches.push_back(std::move(b));
  B2_CATCH
}
int b2_exec_expand(b2_handle child, const b2_handle* projection_programs, int32_t nprojections, b2_handle* out) {
  B2_TRY
  B2_CHECK(nprojections >= 1, "expand needs at least one projection");
  auto* e = new GpuExpandExec();
  e->add_child(exec_from(child));
  e->projections.assign(projection_programs, projection_programs + nprojections);
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_project(b2_handle child, b2_handle program, b2_handle* out) {
  B2_TRY
  auto* e = new GpuProjectExec();
  e->add_child(exec_from(child)); e->program = program;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_hash_aggregate(b2_handle child, b2_handle program, int32_t has_predicate, int32_t mode, const int32_t* keys, int32_t nkeys,
                           const b2_agg_spec* aggs, int32_t naggs, b2_handle* out) {
  B2_TRY
  B2_CHECK(mode == B2_AGG_MODE_PARTIAL || mode == B2_AGG_MODE_FINAL || mode == B2_AGG_MODE_COMPLETE, "unknown aggregate mode");
  std::unique_ptr<GpuHashAggregateExec> e(new GpuHashAggregateExec());
  e->program = mode == B2_AGG_MODE_FINAL ? nullptr : program_from(program);
  e->has_pred = has_predicate != 0; e->mode = mode;
  e->keys.assign(keys, keys + nkeys); e->aggs.assign(aggs, aggs + naggs);
  e->init_counted();
  e->add_child(exec_from(child));
  *out = to_handle(e.release());
  B2_CATCH
}
int b2_exec_aggregate_set_repartitioning(b2_handle agg, int64_t target_bytes, int32_t num_buckets) {
  B2_TRY
  auto* a = dynamic_cast<GpuHashAggregateExec*>(exec_from(agg));
  B2_CHECK(a, "not a hash aggregate node");
  B2_CHECK(target_bytes > 0, "repartitioning: target_bytes must be positive");
  B2_CHECK(num_buckets >= 2 && num_buckets <= 256, "repartitioning: 2 to 256 buckets");
  B2_CHECK(!a->done, "repartitioning must be set before the aggregate runs");
  a->rp_target = target_bytes;
  a->rp_parts = num_buckets;
  B2_CATCH
}
int b2_exec_aggregate_repartition_stats(b2_handle agg, int64_t* out4) {
  B2_TRY
  auto* a = dynamic_cast<GpuHashAggregateExec*>(exec_from(agg));
  B2_CHECK(a, "not a hash aggregate node");
  for (int i = 0; i < 4; i++) out4[i] = a->rp_stats[i];
  B2_CATCH
}
int b2_exec_shuffled_hash_join(b2_handle stream_child, b2_handle build_child, const int32_t* stream_keys, const int32_t* build_keys, int32_t nkeys,
                               int32_t kind, int32_t nulls_equal, b2_handle* out) {
  B2_TRY
  auto* e = new GpuShuffledHashJoinExec();
  e->add_child(exec_from(stream_child)); e->add_child(exec_from(build_child));
  e->stream_keys.assign(stream_keys, stream_keys + nkeys); e->build_keys.assign(build_keys, build_keys + nkeys);
  e->kind = kind; e->nulls_equal = nulls_equal != 0;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_shuffled_hash_join_select(b2_handle stream_child, b2_handle build_child, const int32_t* stream_keys, const int32_t* build_keys, int32_t nkeys,
                                      int32_t kind, int32_t nulls_equal, const int32_t* stream_out, int32_t nstream_out, const int32_t* build_out,
                                      int32_t nbuild_out, b2_handle* out) {
  B2_TRY
  B2_CHECK(nstream_out + nbuild_out >= 1, "join: at least one output column");
  auto* e = new GpuShuffledHashJoinExec();
  e->add_child(exec_from(stream_child)); e->add_child(exec_from(build_child));
  e->stream_keys.assign(stream_keys, stream_keys + nkeys); e->build_keys.assign(build_keys, build_keys + nkeys);
  e->kind = kind; e->nulls_equal = nulls_equal != 0;
  e->pruned = true;
  e->stream_out.assign(stream_out, stream_out + nstream_out); e->build_out.assign(build_out, build_out + nbuild_out);
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_join_set_condition(b2_handle join, b2_handle condition_program) {
  B2_TRY
  auto* j = dynamic_cast<GpuShuffledHashJoinExec*>(exec_from(join));
  B2_CHECK(j, "not a hash join node");
  j->condition = condition_program;
  B2_CATCH
}
int b2_exec_join_set_sub_partitioning(b2_handle join, int64_t target_bytes, int32_t num_partitions) {
  B2_TRY
  auto* j = dynamic_cast<GpuShuffledHashJoinExec*>(exec_from(join));
  B2_CHECK(j, "not a hash join node");
  B2_CHECK(num_partitions >= 2 && num_partitions <= 256, "sub-partitioning: 2 to 256 partitions");
  B2_CHECK(!j->built, "sub-partitioning must be set before the join runs");
  j->sp_target = std::max<int64_t>(target_bytes, 16 << 10);   // at least 16 KiB, like the sort's target
  j->sp_parts = num_partitions;
  B2_CATCH
}
int b2_exec_join_sub_partition_stats(b2_handle join, int64_t* out4) {
  B2_TRY
  auto* j = dynamic_cast<GpuShuffledHashJoinExec*>(exec_from(join));
  B2_CHECK(j, "not a hash join node");
  for (int i = 0; i < 4; i++) out4[i] = j->sp_stats[i];
  B2_CATCH
}
int b2_exec_join_emit_stats(b2_handle join, int64_t* out3) {
  B2_TRY
  auto* j = dynamic_cast<GpuShuffledHashJoinExec*>(exec_from(join));
  B2_CHECK(j, "not a hash join node");
  for (int i = 0; i < 3; i++) out3[i] = j->em_stats[i];
  B2_CATCH
}
int b2_exec_broadcast_exchange(b2_handle child, b2_handle comm, int32_t rank, int32_t world, b2_handle* out) {
  B2_TRY
  auto* e = new GpuBroadcastExchangeExec();
  e->add_child(exec_from(child));
  e->comm = comm; e->rank = rank; e->world = world;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_sort(b2_handle child, const b2_order_by_arg* order, int32_t norder, int32_t global, int64_t limit, b2_handle* out) {
  B2_TRY
  auto* e = new GpuSortExec();
  e->add_child(exec_from(child));
  e->order.assign(order, order + norder); e->global = global != 0; e->limit = limit;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_sort_out_of_core(b2_handle child, const b2_order_by_arg* order, int32_t norder, int64_t target_bytes, b2_handle* out) {
  B2_TRY
  B2_CHECK(norder >= 1 && norder < 16, "out-of-core sort: 1 to 15 sort keys");
  auto* e = new GpuOutOfCoreSortExec();
  e->add_child(exec_from(child));
  e->order.assign(order, order + norder);
  e->target = std::max<int64_t>(target_bytes, 16 << 10);   // GpuSortExec.targetSize: at least 16 KiB
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_coalesce(b2_handle child, int64_t target_rows, b2_handle* out) {
  B2_TRY
  auto* e = new GpuCoalesceBatches();
  e->add_child(exec_from(child)); e->target_rows = target_rows;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_shuffle_exchange(b2_handle child, const int32_t* key_cols, int32_t nkeys, b2_handle comm, int32_t world, b2_handle* out) {
  B2_TRY
  auto* e = new GpuShuffleExchangeExec();
  e->add_child(exec_from(child));
  e->key_cols.assign(key_cols, key_cols + nkeys); e->comm = comm; e->world = world;
  *out = to_handle(e);
  B2_CATCH
}
int b2_exec_next(b2_handle exec, b2_handle* out_table) {
  B2_TRY
  semaphore_acquire_if_necessary();   // GpuSemaphore.acquireIfNecessary: the task enters the GPU at its first batch
  *out_table = to_handle(exec_from(exec)->next());
  B2_CATCH
}
int b2_exec_metrics(b2_handle exec, int64_t* out3) {
  B2_TRY
  GpuExec* e = exec_from(exec);
  out3[0] = e->num_output_rows; out3[1] = e->num_output_batches; out3[2] = e->op_time_ns;
  B2_CATCH
}
int b2_exec_device_time(b2_handle exec, double* out2) {
  B2_TRY
  GpuExec* e = exec_from(exec);
  const double total = GpuExec::span_ms(e->spans), kids = GpuExec::span_ms(e->child_spans);
  out2[0] = total - kids; out2[1] = total;
  B2_CATCH
}
int b2_exec_close(b2_handle exec) {
  B2_TRY
  exec_from(exec)->release();
  B2_CATCH
}

}  // extern "C"
