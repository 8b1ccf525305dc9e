// common.cuh — data model, error plumbing and device-memory helpers shared by every translation
// unit of libb200sql.so.  Host side of the cudf-Java handle convention (SURVEY.md §8b).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <atomic>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>
#include "../../include/b200sql.h"

namespace b2 {

// ---------------------------------------------------------------------------------------------
// errors
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
void set_last_error(const std::string& m);
int translate_exception();  // called inside catch(...)

#define B2_TRY try {
#define B2_CATCH                         \
  }                                      \
  catch (...) {                          \
    return b2::translate_exception();    \
  }                                      \
  return B2_OK;

#define B2_CHECK(cond, msg)                                            \
  do {                                                                 \
    if (!(cond)) throw b2::Error(B2_ERR_INVALID, std::string(msg));    \
  } while (0)

void cuda_check(cudaError_t e, const char* what, const char* file, int line);
#define CUDA_CHECK(x) b2::cuda_check((x), #x, __FILE__, __LINE__)

// ---------------------------------------------------------------------------------------------
// runtime: per-thread stream, stream-ordered pool
cudaStream_t stream();
void* dev_alloc(size_t bytes);            // throws Error(B2_ERR_OOM)
void dev_free(void* p);
void count_launch();
struct KernelTimer {  // scoped CUDA-event timer around a kernel launch; no-op unless profiling is on, or without a name
  void* rec;
  cudaStream_t st;
  explicit KernelTimer(const char* name, cudaStream_t on = nullptr);
  ~KernelTimer();
};
bool profile_enabled();      // b2_profile_enable state
int64_t spill_device(int64_t want_bytes);   // move spillable batches to the host (core.cu); returns device bytes released
void note_retry();
void note_split();
void semaphore_acquire_if_necessary();      // GpuSemaphore.acquireIfNecessary
void semaphore_release_if_necessary();
cudaStream_t aux_stream();   // second per-thread stream for work that may overlap the main stream
int sm_count();

struct DevBuf {  // RAII stream-ordered device buffer
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() {}
  explicit DevBuf(size_t n) : p(n ? dev_alloc(n) : nullptr), bytes(n) {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DevBuf() { reset(); }
  void reset() { if (p) dev_free(p); p = nullptr; bytes = 0; }
  void* release() { void* r = p; p = nullptr; bytes = 0; return r; }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// ---------------------------------------------------------------------------------------------
// types
inline int dtype_width(int dt) {
  switch (dt) {
    case B2_BOOL8: case B2_INT8: return 1;
    case B2_INT16: return 2;
    case B2_INT32: case B2_FLOAT32: case B2_DATE32: case B2_DECIMAL32: return 4;
    case B2_INT64: case B2_FLOAT64: case B2_TIMESTAMP_US: case B2_DECIMAL64: return 8;
    case B2_DECIMAL128: return 16;
    case B2_STRING: return 0;
  }
  throw Error(B2_ERR_INVALID, "unknown dtype " + std::to_string(dt));
}
inline bool is_decimal(int dt) { return dt == B2_DECIMAL32 || dt == B2_DECIMAL64 || dt == B2_DECIMAL128; }
inline bool is_float(int dt) { return dt == B2_FLOAT32 || dt == B2_FLOAT64; }
inline size_t validity_bytes(int64_t rows) {  // 1 bit/row padded to 64 B (GpuBatchUtils.scala:33-41)
  return (size_t)(((rows + 511) / 512) * 64);
}
inline size_t pad64(size_t b) { return (b + 63) & ~(size_t)63; }

// ---------------------------------------------------------------------------------------------
// Column / Table: reference counted, immutable once built
struct Column {
  std::atomic<int> refs{1};
  int dtype = B2_INT64;
  int scale = 0;
  int64_t size = 0;
  int64_t null_count = 0;
  DevBuf data;       // values or chars
  DevBuf valid;      // bitmask or empty
  DevBuf offsets;    // strings
  int64_t chars_bytes = 0;

  const uint32_t* validity() const { return valid.as<uint32_t>(); }
  bool nullable() const { return valid.p != nullptr; }
};

struct Table {
  std::atomic<int> refs{1};
  std::vector<Column*> cols;  // each holds one reference
  int64_t rows = 0;
  ~Table();
};

Column* col_from(b2_handle h);
Table* table_from(b2_handle h);
inline b2_handle to_handle(void* p) { return (b2_handle)(intptr_t)p; }
void col_incref(Column* c);
void col_release(Column* c);
void table_release(Table* t);

// allocate an output column (data + optional validity); data is uninitialised
Column* new_column(int dtype, int scale, int64_t size, bool with_validity);
// make a table taking ownership of the column references
Table* new_table(std::vector<Column*>&& cols);
// device bytes of a table as the spill store counts them: data + validity + offsets
int64_t table_bytes(const Table* t);
// count nulls from the bitmask into col->null_count, dropping the mask if there are none
void finalize_nulls(Column* c);

struct ColGuard {  // releases on scope exit unless released
  Column* c;
  explicit ColGuard(Column* c_) : c(c_) {}
  ~ColGuard() { if (c) col_release(c); }
  Column* release() { Column* r = c; c = nullptr; return r; }
};
struct ColsGuard {
  std::vector<Column*> v;
  ~ColsGuard() { for (auto* c : v) if (c) col_release(c); }
  std::vector<Column*> release() { std::vector<Column*> r; r.swap(v); return r; }
};

// device-side view of a column passed to kernels by value
struct ColView {
  const void* data;
  const uint32_t* valid;   // null when no nulls
  const int32_t* offsets;  // strings
  int32_t dtype;
  int32_t width;
};
inline ColView view_of(const Column* c) {
  ColView v;
  v.data = c->data.p; v.valid = c->validity(); v.offsets = c->offsets.as<int32_t>();
  v.dtype = c->dtype; v.width = dtype_width(c->dtype);
  return v;
}

// Descriptor-sized uploads (page tables, programs, plans) do not use the DMA engine: it serves copies in issue
// order, so a 100-byte upload would wait behind the next batch's 0.5 GB file copy.  The bytes are staged in a
// mapped pinned ring and pulled over by a small kernel on the compute stream (core.cu).
void h2d_bytes(void* dst, const void* src, size_t bytes);
template <typename T>
inline void h2d(void* dst, const T* src, size_t n) { h2d_bytes(dst, src, n * sizeof(T)); }
template <typename T>
inline void d2h(T* dst, const void* src, size_t n) {
  CUDA_CHECK(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, stream()));
}
inline void sync() { CUDA_CHECK(cudaStreamSynchronize(stream())); }

inline int grid_for(int64_t work_items, int per_block, int ctas_per_sm = 8) {
  int64_t need = (work_items + per_block - 1) / per_block;
  int64_t cap = (int64_t)sm_count() * ctas_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

}  // namespace b2

// ---------------------------------------------------------------------------------------------
// device helpers
#ifdef __CUDACC__
namespace b2 {
__device__ __forceinline__ bool bit_get(const uint32_t* m, int64_t i) {
  return (m[i >> 5] >> (i & 31)) & 1u;
}
__device__ __forceinline__ bool row_valid(const uint32_t* m, int64_t i) {
  return m == nullptr || bit_get(m, i);
}

// Every kernel launch of the library goes through launch(), so each one is checked and counted the same way.
// A launch asking for more dynamic shared memory than the kernel's limit first raises the limit (core.cu).
void reserve_dyn_smem(const void* kernel, size_t smem);
// Raises a rejected launch as an Error naming the kernel; counts the launch otherwise (core.cu).
void launch_done(const void* kernel);

// Named form: `timer` (may be null) times exactly this launch when profiling is on.
template <typename... P, typename... A>
inline void launch(const char* timer, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  if (smem) reserve_dyn_smem((const void*)kernel, smem);
  {
    KernelTimer kt(timer, st);
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
  }
  launch_done((const void*)kernel);
}
template <typename... P, typename... A>
inline void launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  launch(nullptr, kernel, grid, block, smem, st, std::forward<A>(args)...);
}
typedef __int128 i128;
typedef unsigned __int128 u128;
}  // namespace b2
#endif
