// core.cu — runtime (device init, stream-ordered pool, per-thread stream), column/table handles,
// host<->device transfer, events.  Reference counterparts: GpuDeviceManager.scala:349-445
// (Rmm.initialize, ASYNC allocator mode), GpuColumnVector.java:621-660, HostColumnarToGpu.scala,
// GpuColumnarToRowExec.scala:337-384 (copyToHost).
#include <mutex>
#include <condition_variable>
#include <list>
#include <algorithm>
#include <unordered_map>
#include <cstdio>
#include <cstdlib>
#include <cxxabi.h>
#include "common.cuh"

namespace b2 {

static thread_local std::string g_err;
void set_last_error(const std::string& m) { g_err = m; }

int translate_exception() {
  try {
    throw;
  } catch (const Error& e) {
    g_err = e.what();
    return e.code;
  } catch (const std::bad_alloc& e) {
    g_err = "host allocation failed";
    return B2_ERR_INVALID;
  } catch (const std::exception& e) {
    g_err = e.what();
    return B2_ERR_INVALID;
  } catch (...) {
    g_err = "unknown error";
    return B2_ERR_FATAL;
  }
}

void cuda_check(cudaError_t e, const char* what, const char* file, int line) {
  if (e == cudaSuccess) return;
  std::string m = std::string(cudaGetErrorName(e)) + ": " + cudaGetErrorString(e) + " at " + file +
                  ":" + std::to_string(line) + " (" + what + ")";
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    throw Error(B2_ERR_OOM, m);
  }
  // sticky errors poison the context: the reference exits the executor (Plugin.scala:823-848)
  bool fatal = (e == cudaErrorIllegalAddress || e == cudaErrorLaunchFailure ||
                e == cudaErrorHardwareStackError || e == cudaErrorIllegalInstruction ||
                e == cudaErrorMisalignedAddress || e == cudaErrorECCUncorrectable);
  throw Error(fatal ? B2_ERR_FATAL : B2_ERR_CUDA, m);
}

// ---------------------------------------------------------------------------------------------
static std::mutex g_mu;
static bool g_inited = false;
static int g_device = 0;
static int g_sms = 132;
static std::atomic<int64_t> g_in_use{0};
static std::atomic<int64_t> g_limit{0};
static std::atomic<int64_t> g_launches{0};
static std::unordered_map<void*, size_t> g_sizes;
static thread_local cudaStream_t t_stream = nullptr;
static thread_local bool t_stream_owned = false;

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

struct ProfRec { const char* name; cudaEvent_t a, b; };
static std::atomic<bool> g_prof{false};
static std::mutex g_prof_mu;
static std::vector<ProfRec*> g_prof_recs;
KernelTimer::KernelTimer(const char* name, cudaStream_t on) : rec(nullptr), st(on) {
  if (!name || !g_prof.load(std::memory_order_relaxed)) return;
  if (!st) st = stream();
  ProfRec* r = new ProfRec();
  r->name = name;
  cudaEventCreate(&r->a); cudaEventCreate(&r->b);
  cudaEventRecord(r->a, st);
  rec = r;
}
KernelTimer::~KernelTimer() {
  if (!rec) return;
  ProfRec* r = reinterpret_cast<ProfRec*>(rec);
  cudaEventRecord(r->b, st);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_recs.push_back(r);
}
// The limit is per kernel and only ever raised, under one lock, so a thread launching with less shared memory
// can never lower it between another thread's raise and launch.  A kernel starts out allowed 48 KB of shared
// memory in all, static included; the first launch with dynamic shared memory reads both once.
void reserve_dyn_smem(const void* kernel, size_t smem) {
  static std::mutex mu;
  static std::unordered_map<const void*, size_t> limit;   // kernel -> dynamic shared memory it may launch with
  std::lock_guard<std::mutex> lk(mu);
  auto it = limit.find(kernel);
  if (it == limit.end()) {
    cudaFuncAttributes a;
    CUDA_CHECK(cudaFuncGetAttributes(&a, kernel));
    const size_t dflt = a.sharedSizeBytes < 48 * 1024 ? 48 * 1024 - a.sharedSizeBytes : 0;
    it = limit.emplace(kernel, std::min<size_t>(dflt, (size_t)a.maxDynamicSharedSizeBytes)).first;
  }
  if (smem <= it->second) return;
  CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  it->second = smem;
}

void launch_done(const void* kernel) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    std::string what = "launch of ";
    const char* name = nullptr;
    if (cudaFuncGetName(&name, kernel) == cudaSuccess && name) {
      int st = 0;
      char* dm = abi::__cxa_demangle(name, nullptr, nullptr, &st);
      what += st == 0 && dm ? dm : name;
      free(dm);
    } else {
      cudaGetLastError();   // the failed lookup must not surface at a later, unrelated check
      what += "a kernel";
    }
    cuda_check(e, what.c_str(), __FILE__, __LINE__);
  }
  count_launch();
}

int sm_count() { return g_sms; }
bool profile_enabled() { return g_prof.load(std::memory_order_relaxed); }

static void ensure_init() {
  if (g_inited) return;
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_inited) return;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    throw Error(B2_ERR_CUDA, "libb200sql: no CUDA device available (this library has no CPU fallback)");
  }
  CUDA_CHECK(cudaGetDevice(&g_device));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, g_device));
  g_sms = prop.multiProcessorCount;
  cudaMemPool_t pool;
  CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, g_device));
  uint64_t thr = UINT64_MAX;  // keep freed memory in the pool: Rmm pool behaviour
  CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
  g_inited = true;
}

static thread_local cudaStream_t t_aux = nullptr;
cudaStream_t aux_stream() {
  if (!t_aux) { stream(); CUDA_CHECK(cudaStreamCreateWithFlags(&t_aux, cudaStreamNonBlocking)); }
  return t_aux;
}

cudaStream_t stream() {
  if (!t_stream) {
    ensure_init();
    CUDA_CHECK(cudaSetDevice(g_device));
    CUDA_CHECK(cudaStreamCreateWithFlags(&t_stream, cudaStreamNonBlocking));
    t_stream_owned = true;
  }
  return t_stream;
}

// ---- staged descriptor uploads ------------------------------------------------------------------------------
static constexpr size_t STAGE_BYTES = 32u << 20, STAGE_MAX = 4u << 20;
struct StageRing {
  char* host = nullptr; char* dev = nullptr; size_t head = 0;
  cudaEvent_t half[2] = {nullptr, nullptr};   // recorded after the last reader of each half
  bool armed[2] = {false, false};
};
static thread_local StageRing t_stage;

__global__ void stage_pull_kernel(char* dst, const char* src, size_t bytes) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {
    const size_t n16 = bytes >> 4;
    for (size_t i = i0; i < n16; i += step) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    for (size_t i = (n16 << 4) + i0; i < bytes; i += step) dst[i] = src[i];
  } else {
    for (size_t i = i0; i < bytes; i += step) dst[i] = src[i];
  }
}

void h2d_bytes(void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return;
  cudaStream_t s = stream();
  if (bytes > STAGE_MAX) { CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s)); return; }
  StageRing& r = t_stage;
  if (!r.host) {
    CUDA_CHECK(cudaHostAlloc((void**)&r.host, STAGE_BYTES, cudaHostAllocMapped));
    CUDA_CHECK(cudaHostGetDevicePointer((void**)&r.dev, r.host, 0));
    for (int i = 0; i < 2; i++) CUDA_CHECK(cudaEventCreateWithFlags(&r.half[i], cudaEventDisableTiming | cudaEventBlockingSync));
  }
  const size_t half = STAGE_BYTES / 2, need = (bytes + 15) & ~size_t(15);
  size_t at = r.head;
  int h = (int)std::min<size_t>(1, at / half);
  if (at + need > (size_t)(h + 1) * half) {          // does not fit in the rest of this half: close it, move on
    CUDA_CHECK(cudaEventRecord(r.half[h], s)); r.armed[h] = true;
    h ^= 1; at = (size_t)h * half;
    if (r.armed[h]) { CUDA_CHECK(cudaEventSynchronize(r.half[h])); r.armed[h] = false; }
  }
  memcpy(r.host + at, src, bytes);
  r.head = at + need;
  const int threads = 256;
  const int blocks = (int)std::min<size_t>(64, (bytes / 16 + threads - 1) / threads + 1);
  launch("stage_pull_kernel", stage_pull_kernel, blocks, threads, 0, s, (char*)dst, r.dev + at, bytes);
}

int64_t spill_device(int64_t want_bytes);   // below: the spill store

void* dev_alloc(size_t bytes) {
  if (bytes == 0) bytes = 64;
  bytes = pad64(bytes);
  int64_t lim = g_limit.load();
  if (lim > 0 && g_in_use.load() + (int64_t)bytes > lim) {
    // DeviceMemoryEventHandler.onAllocFailure (DeviceMemoryEventHandler.scala): spill first, fail with a retryable OOM if that was not enough
    spill_device(g_in_use.load() + (int64_t)bytes - lim);
    if (g_in_use.load() + (int64_t)bytes > lim)
      throw Error(B2_ERR_OOM, "allocation of " + std::to_string(bytes) + " B exceeds the configured limit");
  }
  void* p = nullptr;
  cudaStream_t s = stream();
  cudaError_t e = cudaMallocAsync(&p, bytes, s);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    // give outstanding frees a chance to land and move spillable batches to the host, then retry once
    spill_device((int64_t)bytes);
    cudaDeviceSynchronize();
    e = cudaMallocAsync(&p, bytes, s);
  }
  if (e != cudaSuccess) cuda_check(e, ("cudaMallocAsync of " + std::to_string(bytes) + " B with " + std::to_string(g_in_use.load()) + " B in use").c_str(), __FILE__, __LINE__);
  g_in_use.fetch_add((int64_t)bytes);
  {
    std::lock_guard<std::mutex> lk(g_mu);
    g_sizes[p] = bytes;
  }
  return p;
}

void dev_free(void* p) {
  if (!p) return;
  size_t bytes = 0;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_sizes.find(p);
    if (it != g_sizes.end()) { bytes = it->second; g_sizes.erase(it); }
  }
  g_in_use.fetch_sub((int64_t)bytes);
  cudaFreeAsync(p, stream());
}


// ---------------------------------------------------------------------------------------------
// (f4) memory pressure: spill store, semaphore, retry accounting.
// Reference: spill/SpillFramework.scala:49-150 (SpillableColumnarBatch handles: anything held across iterator next() calls
// may be moved to host memory at any time and is brought back on access), DeviceMemoryEventHandler (spill on allocation
// failure, then GpuRetryOOM), GpuSemaphore.scala:183-260 (bounded number of tasks on the GPU), RmmRapidsRetryIterator.scala:
// 65-203 (withRetry / split-and-retry: implemented in exec.cu above this store).
struct SpilledColumn {   // (distinct name: exec.cu has its own HostColumn; two layouts under one name would be an ODR violation)
  int dtype = 0, scale = 0; int64_t size = 0, null_count = 0, chars_bytes = 0;
  std::vector<uint8_t> data, valid, offsets;
};
struct Spillable {
  std::mutex mu;
  Table* dev = nullptr;              // resident form (one reference held by the store)
  std::vector<SpilledColumn> host;      // spilled form
  int64_t bytes = 0;
  uint64_t last_use = 0;
};
static std::mutex g_spill_mu;
static std::list<Spillable*> g_spillables;
static std::atomic<uint64_t> g_use_clock{1};
static std::atomic<int64_t> g_spilled_bytes{0}, g_unspilled_bytes{0}, g_retries{0}, g_splits{0};
void note_retry() { g_retries.fetch_add(1); }
void note_split() { g_splits.fetch_add(1); }

int64_t table_bytes(const Table* t) {
  int64_t b = 0;
  for (auto* c : t->cols) b += (int64_t)c->data.bytes + (int64_t)c->valid.bytes + (int64_t)c->offsets.bytes;
  return b;
}
static bool spill_one(Spillable* sp) {   // sp->mu held; true when device memory was released
  if (!sp->dev || sp->dev->refs.load() != 1) return false;   // somebody is using the batch right now
  for (auto* c : sp->dev->cols) if (c->refs.load() != 1) return false;
  cudaStream_t s = stream();
  sp->host.clear();
  for (auto* c : sp->dev->cols) {
    SpilledColumn h;
    h.dtype = c->dtype; h.scale = c->scale; h.size = c->size; h.null_count = c->null_count; h.chars_bytes = c->chars_bytes;
    const size_t db = c->dtype == B2_STRING ? (size_t)c->chars_bytes : (size_t)c->size * dtype_width(c->dtype);
    h.data.resize(db);
    if (db) CUDA_CHECK(cudaMemcpyAsync(h.data.data(), c->data.p, db, cudaMemcpyDeviceToHost, s));
    if (c->valid.p) { h.valid.resize(validity_bytes(c->size)); CUDA_CHECK(cudaMemcpyAsync(h.valid.data(), c->valid.p, h.valid.size(), cudaMemcpyDeviceToHost, s)); }
    if (c->dtype == B2_STRING) { h.offsets.resize((size_t)(c->size + 1) * 4); CUDA_CHECK(cudaMemcpyAsync(h.offsets.data(), c->offsets.p, h.offsets.size(), cudaMemcpyDeviceToHost, s)); }
    sp->host.push_back(std::move(h));
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  table_release(sp->dev);
  sp->dev = nullptr;
  g_spilled_bytes.fetch_add(sp->bytes);
  return true;
}
// move least-recently-used spillable batches to the host until `want_bytes` of device memory were released
int64_t spill_device(int64_t want_bytes) {
  std::vector<Spillable*> order;
  {
    std::lock_guard<std::mutex> lk(g_spill_mu);
    order.assign(g_spillables.begin(), g_spillables.end());
  }
  std::sort(order.begin(), order.end(), [](Spillable* a, Spillable* b) { return a->last_use < b->last_use; });
  int64_t freed = 0;
  for (auto* sp : order) {
    if (freed >= want_bytes) break;
    std::unique_lock<std::mutex> lk(sp->mu, std::try_to_lock);
    if (!lk.owns_lock()) continue;
    if (spill_one(sp)) freed += sp->bytes;
  }
  return freed;
}
static Table* unspill(Spillable* sp) {   // sp->mu held
  ColsGuard cols;
  cudaStream_t s = stream();
  for (auto& h : sp->host) {
    std::unique_ptr<Column> c(new Column());
    c->dtype = h.dtype; c->scale = h.scale; c->size = h.size; c->null_count = h.null_count; c->chars_bytes = h.chars_bytes;
    c->data = DevBuf(h.data.size());
    if (!h.data.empty()) CUDA_CHECK(cudaMemcpyAsync(c->data.p, h.data.data(), h.data.size(), cudaMemcpyHostToDevice, s));
    if (!h.valid.empty()) { c->valid = DevBuf(h.valid.size()); CUDA_CHECK(cudaMemcpyAsync(c->valid.p, h.valid.data(), h.valid.size(), cudaMemcpyHostToDevice, s)); }
    if (!h.offsets.empty()) { c->offsets = DevBuf(h.offsets.size()); CUDA_CHECK(cudaMemcpyAsync(c->offsets.p, h.offsets.data(), h.offsets.size(), cudaMemcpyHostToDevice, s)); }
    cols.v.push_back(c.release());
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  sp->host.clear(); sp->host.shrink_to_fit();
  g_unspilled_bytes.fetch_add(sp->bytes);
  return new_table(cols.release());
}

// GpuSemaphore: at most `permits` threads (tasks) between acquire and release; 0 = unlimited
static std::mutex g_sem_mu;
static std::condition_variable g_sem_cv;
static int g_sem_permits = 0, g_sem_in_use = 0;
static int64_t g_sem_waits = 0;
static thread_local bool t_sem_held = false;
void semaphore_acquire_if_necessary() {
  if (t_sem_held) return;
  std::unique_lock<std::mutex> lk(g_sem_mu);
  if (g_sem_permits <= 0) return;   // unlimited: nothing to account for
  if (g_sem_in_use >= g_sem_permits) g_sem_waits++;
  g_sem_cv.wait(lk, [] { return g_sem_permits <= 0 || g_sem_in_use < g_sem_permits; });
  if (g_sem_permits <= 0) return;   // the limit was lifted while waiting
  g_sem_in_use++;
  t_sem_held = true;
}
void semaphore_release_if_necessary() {
  if (!t_sem_held) return;
  { std::lock_guard<std::mutex> lk(g_sem_mu); if (g_sem_in_use > 0) g_sem_in_use--; }
  t_sem_held = false;
  g_sem_cv.notify_one();
}

// ---------------------------------------------------------------------------------------------
Table::~Table() {
  for (auto* c : cols) if (c) col_release(c);
}
Column* col_from(b2_handle h) {
  if (h == 0) throw Error(B2_ERR_INVALID, "null column handle");
  return reinterpret_cast<Column*>((intptr_t)h);
}
Table* table_from(b2_handle h) {
  if (h == 0) throw Error(B2_ERR_INVALID, "null table handle");
  return reinterpret_cast<Table*>((intptr_t)h);
}
void col_incref(Column* c) { c->refs.fetch_add(1); }
void col_release(Column* c) {
  if (c->refs.fetch_sub(1) == 1) delete c;
}
void table_release(Table* t) {
  if (t->refs.fetch_sub(1) == 1) delete t;
}

Column* new_column(int dtype, int scale, int64_t size, bool with_validity) {
  if (size > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "column of " + std::to_string(size) + " rows");
  std::unique_ptr<Column> c(new Column());
  c->dtype = dtype; c->scale = scale; c->size = size;
  int w = dtype_width(dtype);
  if (w > 0) c->data = DevBuf((size_t)size * w);
  if (with_validity) c->valid = DevBuf(validity_bytes(size));
  c->null_count = with_validity ? -1 : 0;
  return c.release();
}

Table* new_table(std::vector<Column*>&& cols) {
  Table* t = new Table();
  t->cols = std::move(cols);
  t->rows = t->cols.empty() ? 0 : t->cols[0]->size;
  for (auto* c : t->cols)
    if (c->size != t->rows) { delete t; throw Error(B2_ERR_INVALID, "table columns differ in length"); }
  return t;
}

__global__ void count_valid_kernel(const uint32_t* __restrict__ m, int64_t rows, unsigned long long* out) {
  int64_t words = (rows + 31) >> 5;
  unsigned long long acc = 0;
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < words; w += (int64_t)gridDim.x * blockDim.x) {
    uint32_t v = m[w];
    if (w == words - 1 && (rows & 31)) v &= (1u << (rows & 31)) - 1u;
    acc += __popc(v);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

static int64_t count_nulls(Column* c) {
  if (!c->valid.p) return 0;
  if (c->size == 0) return 0;
  DevBuf cnt(8);
  CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, 8, stream()));
  int64_t words = (c->size + 31) >> 5;
  launch(count_valid_kernel, grid_for(words, 256), 256, 0, stream(), c->validity(), c->size, cnt.as<unsigned long long>());
  unsigned long long h = 0;
  d2h(&h, cnt.p, 1);
  sync();
  return c->size - (int64_t)h;
}

void finalize_nulls(Column* c) {
  if (c->null_count < 0) c->null_count = count_nulls(c);
}

__global__ void fill_kernel(uint8_t* out, int64_t n, int width, uint4 v) {
  const uint8_t* src = reinterpret_cast<const uint8_t*>(&v);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    for (int b = 0; b < width; b++) out[i * width + b] = src[b];
}

}  // namespace b2

using namespace b2;

extern "C" {

const char* b2_last_error(void) { return g_err.c_str(); }
const char* b2_version(void) { return "b200sql 0.1 (sm_90a)"; }

int b2_init(int device, size_t pool_bytes) {
  B2_TRY
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    throw Error(B2_ERR_CUDA, "libb200sql: no CUDA device available (this library has no CPU fallback)");
  }
  B2_CHECK(device >= 0 && device < ndev, "bad device ordinal");
  CUDA_CHECK(cudaSetDevice(device));
  ensure_init();
  g_device = device;
  if (pool_bytes) {  // pre-warm the pool like Rmm.initialize(pool size)
    void* p = nullptr;
    if (cudaMallocAsync(&p, pool_bytes, stream()) == cudaSuccess) cudaFreeAsync(p, stream());
    else cudaGetLastError();
    sync();
  }
  B2_CATCH
}

int b2_shutdown(void) {
  B2_TRY
  if (t_stream && t_stream_owned) { cudaStreamSynchronize(t_stream); cudaStreamDestroy(t_stream); }
  t_stream = nullptr;
  B2_CATCH
}

int b2_stream_sync(void) {
  B2_TRY
  sync();
  B2_CATCH
}

int b2_set_stream(void* s) {
  B2_TRY
  ensure_init();
  if (t_stream && t_stream_owned) { cudaStreamSynchronize(t_stream); cudaStreamDestroy(t_stream); }
  t_stream = (cudaStream_t)s;
  t_stream_owned = false;
  B2_CATCH
}

void* b2_get_stream(void) {
  try { return (void*)stream(); } catch (...) { translate_exception(); return nullptr; }
}

int b2_device_bytes_in_use(int64_t* out) { *out = g_in_use.load(); return B2_OK; }
int b2_set_alloc_limit(int64_t bytes) { g_limit.store(bytes); return B2_OK; }
int b2_kernel_launch_count(int64_t* out) { *out = g_launches.load(); return B2_OK; }

static Column* column_build(int32_t dtype, int32_t scale, int64_t size, const void* data,
                            const void* validity, const int32_t* offsets, cudaMemcpyKind kind) {
  B2_CHECK(size >= 0, "negative size");
  if (size > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "too many rows");
  std::unique_ptr<Column> c(new Column());
  c->dtype = dtype; c->scale = scale; c->size = size;
  int w = dtype_width(dtype);
  cudaStream_t s = stream();
  if (dtype == B2_STRING) {
    B2_CHECK(offsets != nullptr || size == 0, "string column needs offsets");
    c->offsets = DevBuf((size_t)(size + 1) * 4);
    int32_t nchars = 0;
    if (size > 0) {
      CUDA_CHECK(cudaMemcpyAsync(c->offsets.p, offsets, (size_t)(size + 1) * 4, kind, s));
      if (kind == cudaMemcpyHostToDevice) nchars = offsets[size];
      else { d2h(&nchars, (const char*)c->offsets.p + size * 4, 1); sync(); }
    } else {
      CUDA_CHECK(cudaMemsetAsync(c->offsets.p, 0, 4, s));
    }
    c->chars_bytes = nchars;
    c->data = DevBuf((size_t)nchars);
    if (nchars) CUDA_CHECK(cudaMemcpyAsync(c->data.p, data, (size_t)nchars, kind, s));
  } else {
    c->data = DevBuf((size_t)size * w);
    if (size) CUDA_CHECK(cudaMemcpyAsync(c->data.p, data, (size_t)size * w, kind, s));
  }
  if (validity) {
    size_t vb = validity_bytes(size);
    c->valid = DevBuf(vb);
    CUDA_CHECK(cudaMemsetAsync(c->valid.p, 0, vb, s));
    CUDA_CHECK(cudaMemcpyAsync(c->valid.p, validity, (size_t)((size + 7) / 8), kind, s));
    c->null_count = -1;
  }
  if (kind == cudaMemcpyHostToDevice) sync();  // the caller may free its host buffers on return
  return c.release();
}

int b2_column_from_host(int32_t dtype, int32_t scale, int64_t size, const void* data,
                        const uint8_t* validity_bits, const int32_t* offsets, b2_handle* out) {
  B2_TRY
  *out = to_handle(column_build(dtype, scale, size, data, validity_bits, offsets, cudaMemcpyHostToDevice));
  B2_CATCH
}

int b2_column_from_device(int32_t dtype, int32_t scale, int64_t size, const void* data,
                          const uint32_t* validity_bits, const int32_t* offsets, b2_handle* out) {
  B2_TRY
  *out = to_handle(column_build(dtype, scale, size, data, validity_bits, offsets, cudaMemcpyDeviceToDevice));
  B2_CATCH
}

int b2_column_info_get(b2_handle h, b2_column_info* out) {
  B2_TRY
  Column* c = col_from(h);
  finalize_nulls(c);
  out->dtype = c->dtype; out->scale = c->scale; out->size = c->size; out->null_count = c->null_count;
  out->data = c->data.p; out->validity = c->validity(); out->offsets = c->offsets.as<int32_t>();
  out->data_bytes = c->dtype == B2_STRING ? c->chars_bytes : c->size * dtype_width(c->dtype);
  B2_CATCH
}

int b2_column_to_host(b2_handle h, void* data, uint8_t* validity_bits, int32_t* offsets) {
  B2_TRY
  Column* c = col_from(h);
  cudaStream_t s = stream();
  if (c->dtype == B2_STRING) {
    if (offsets) CUDA_CHECK(cudaMemcpyAsync(offsets, c->offsets.p, (size_t)(c->size + 1) * 4, cudaMemcpyDeviceToHost, s));
    if (data && c->chars_bytes) CUDA_CHECK(cudaMemcpyAsync(data, c->data.p, (size_t)c->chars_bytes, cudaMemcpyDeviceToHost, s));
  } else if (data && c->size) {
    CUDA_CHECK(cudaMemcpyAsync(data, c->data.p, (size_t)c->size * dtype_width(c->dtype), cudaMemcpyDeviceToHost, s));
  }
  if (validity_bits) {
    size_t nb = (size_t)((c->size + 7) / 8);
    if (c->valid.p) CUDA_CHECK(cudaMemcpyAsync(validity_bits, c->valid.p, nb, cudaMemcpyDeviceToHost, s));
    else memset(validity_bits, 0xff, nb);
  }
  sync();
  B2_CATCH
}

int b2_column_incref(b2_handle h) {
  B2_TRY
  col_incref(col_from(h));
  B2_CATCH
}
int b2_column_close(b2_handle h) {
  B2_TRY
  col_release(col_from(h));
  B2_CATCH
}

int b2_column_from_scalar(int32_t dtype, int32_t scale, int64_t size, const void* value16,
                          int32_t is_valid, b2_handle* out) {
  B2_TRY
  B2_CHECK(dtype != B2_STRING, "string scalars not supported here");
  ColGuard g(new_column(dtype, scale, size, !is_valid));
  uint4 v = {0, 0, 0, 0};
  if (value16) memcpy(&v, value16, 16);
  if (size) launch(fill_kernel, grid_for(size, 256), 256, 0, stream(), g.c->data.as<uint8_t>(), size, dtype_width(dtype), v);
  if (!is_valid) {
    CUDA_CHECK(cudaMemsetAsync(g.c->valid.p, 0, g.c->valid.bytes, stream()));
    g.c->null_count = size;
  }
  *out = to_handle(g.release());
  B2_CATCH
}

int b2_table_create(const b2_handle* cols, int32_t ncols, b2_handle* out) {
  B2_TRY
  std::vector<Column*> v;
  for (int i = 0; i < ncols; i++) v.push_back(col_from(cols[i]));
  for (auto* c : v) col_incref(c);
  *out = to_handle(new_table(std::move(v)));
  B2_CATCH
}
int b2_table_num_rows(b2_handle t, int64_t* out) {
  B2_TRY
  *out = table_from(t)->rows;
  B2_CATCH
}
int b2_table_num_columns(b2_handle t, int32_t* out) {
  B2_TRY
  *out = (int32_t)table_from(t)->cols.size();
  B2_CATCH
}
int b2_table_column(b2_handle t, int32_t i, b2_handle* out) {
  B2_TRY
  Table* tb = table_from(t);
  B2_CHECK(i >= 0 && i < (int)tb->cols.size(), "column index out of range");
  col_incref(tb->cols[i]);
  *out = to_handle(tb->cols[i]);
  B2_CATCH
}
int b2_table_incref(b2_handle t) {
  B2_TRY
  table_from(t)->refs.fetch_add(1);
  B2_CATCH
}
int b2_table_close(b2_handle t) {
  B2_TRY
  table_release(table_from(t));
  B2_CATCH
}

int b2_profile_enable(int32_t on) {
  B2_TRY
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto* r : g_prof_recs) { cudaEventDestroy(r->a); cudaEventDestroy(r->b); delete r; }
  g_prof_recs.clear();
  g_prof.store(on != 0);
  B2_CATCH
}
int b2_profile_report(char* buf, int64_t capacity) {
  B2_TRY
  sync();
  std::lock_guard<std::mutex> lk(g_prof_mu);
  std::vector<std::string> names; std::vector<double> ms; std::vector<int64_t> cnt;
  for (auto* r : g_prof_recs) {
    float t = 0;
    cudaEventSynchronize(r->b);
    cudaEventElapsedTime(&t, r->a, r->b);
    size_t k = 0;
    for (; k < names.size(); k++) if (names[k] == r->name) break;
    if (k == names.size()) { names.push_back(r->name); ms.push_back(0); cnt.push_back(0); }
    ms[k] += t; cnt[k] += 1;
  }
  std::string out = "[";
  for (size_t k = 0; k < names.size(); k++) {
    char line[256];
    snprintf(line, sizeof(line), "%s{\"name\":\"%s\",\"launches\":%lld,\"ms\":%.6f}", k ? "," : "", names[k].c_str(), (long long)cnt[k], ms[k]);
    out += line;
  }
  out += "]";
  B2_CHECK((int64_t)out.size() + 1 <= capacity, "profile buffer too small");
  memcpy(buf, out.c_str(), out.size() + 1);
  B2_CATCH
}
int b2_host_register(void* ptr, int64_t bytes) {
  B2_TRY
  stream();
  CUDA_CHECK(cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterDefault));
  B2_CATCH
}
int b2_host_unregister(void* ptr) {
  B2_TRY
  CUDA_CHECK(cudaHostUnregister(ptr));
  B2_CATCH
}
int b2_device_alloc(int64_t bytes, void** out) {
  B2_TRY
  *out = dev_alloc((size_t)bytes);
  B2_CATCH
}
int b2_device_free(void* ptr) {
  B2_TRY
  dev_free(ptr);
  B2_CATCH
}
int b2_memcpy_h2d(void* dst, const void* src, int64_t bytes) {
  B2_TRY
  CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyHostToDevice, stream()));
  sync();
  B2_CATCH
}

struct Upload { void* dev; size_t bytes; cudaEvent_t done; };
static thread_local cudaStream_t t_copy = nullptr;
int b2_upload_start(const void* pinned_host, int64_t bytes, b2_handle* out_upload) {
  B2_TRY
  stream();
  if (!t_copy) CUDA_CHECK(cudaStreamCreateWithFlags(&t_copy, cudaStreamNonBlocking));
  std::unique_ptr<Upload> u(new Upload());
  u->bytes = (size_t)bytes + 64;
  CUDA_CHECK(cudaMallocAsync(&u->dev, u->bytes, t_copy));
  // in 8 MB pieces: the DMA engine serves work items in order, and the decode of the batch in flight issues
  // small descriptor uploads that must not queue behind one 0.5 GB copy
  const size_t piece = 8u << 20;
  for (size_t off = 0; off < (size_t)bytes; off += piece)
    CUDA_CHECK(cudaMemcpyAsync((char*)u->dev + off, (const char*)pinned_host + off, std::min(piece, (size_t)bytes - off), cudaMemcpyHostToDevice, t_copy));
  CUDA_CHECK(cudaEventCreateWithFlags(&u->done, cudaEventDisableTiming));
  CUDA_CHECK(cudaEventRecord(u->done, t_copy));
  *out_upload = to_handle(u.release());
  B2_CATCH
}
int b2_upload_wait(b2_handle upload, void** out_device_ptr) {
  B2_TRY
  Upload* u = reinterpret_cast<Upload*>((intptr_t)upload);
  CUDA_CHECK(cudaStreamWaitEvent(stream(), u->done, 0));
  *out_device_ptr = u->dev;
  B2_CATCH
}
int b2_upload_free(b2_handle upload) {
  B2_TRY
  Upload* u = reinterpret_cast<Upload*>((intptr_t)upload);
  cudaFreeAsync(u->dev, stream());   // after everything queued on the compute stream that read it
  cudaEventDestroy(u->done);
  delete u;
  B2_CATCH
}


// ---- (f4) spill store / semaphore / retry accounting ---------------------------------------------------------------------------
int b2_spillable_create(b2_handle table, b2_handle* out) {
  B2_TRY
  Table* t = table_from(table);
  std::unique_ptr<Spillable> sp(new Spillable());
  t->refs.fetch_add(1);
  for (auto* c : t->cols) finalize_nulls(c);
  sp->dev = t; sp->bytes = table_bytes(t); sp->last_use = g_use_clock.fetch_add(1);
  {
    std::lock_guard<std::mutex> lk(g_spill_mu);
    g_spillables.push_back(sp.get());
  }
  *out = to_handle(sp.release());
  B2_CATCH
}
int b2_spillable_get(b2_handle h, b2_handle* out_table) {
  B2_TRY
  B2_CHECK(h, "null spillable handle");
  Spillable* sp = reinterpret_cast<Spillable*>((intptr_t)h);
  std::lock_guard<std::mutex> lk(sp->mu);
  if (!sp->dev) sp->dev = unspill(sp);
  sp->last_use = g_use_clock.fetch_add(1);
  sp->dev->refs.fetch_add(1);
  *out_table = to_handle(sp->dev);
  B2_CATCH
}
int b2_spillable_is_spilled(b2_handle h, int32_t* out) {
  B2_TRY
  B2_CHECK(h, "null spillable handle");
  Spillable* sp = reinterpret_cast<Spillable*>((intptr_t)h);
  std::lock_guard<std::mutex> lk(sp->mu);
  *out = sp->dev ? 0 : 1;
  B2_CATCH
}
int b2_spillable_close(b2_handle h) {
  B2_TRY
  B2_CHECK(h, "null spillable handle");
  Spillable* sp = reinterpret_cast<Spillable*>((intptr_t)h);
  {
    std::lock_guard<std::mutex> lk(g_spill_mu);
    g_spillables.remove(sp);
  }
  { std::lock_guard<std::mutex> lk(sp->mu); if (sp->dev) table_release(sp->dev); sp->dev = nullptr; }
  delete sp;
  B2_CATCH
}
int b2_spill(int64_t want_bytes, int64_t* out_freed) {
  B2_TRY
  *out_freed = spill_device(want_bytes);
  B2_CATCH
}
int b2_memory_stats(int64_t* out6) {
  out6[0] = g_in_use.load(); out6[1] = g_limit.load(); out6[2] = g_spilled_bytes.load(); out6[3] = g_unspilled_bytes.load();
  out6[4] = g_retries.load(); out6[5] = g_splits.load();
  return B2_OK;
}
int b2_semaphore_init(int32_t permits) {
  std::lock_guard<std::mutex> lk(g_sem_mu);
  g_sem_permits = permits;
  if (permits <= 0) g_sem_in_use = 0;
  g_sem_cv.notify_all();
  return B2_OK;
}
int b2_semaphore_acquire(void) { semaphore_acquire_if_necessary(); return B2_OK; }
int b2_semaphore_release(void) { semaphore_release_if_necessary(); return B2_OK; }
int b2_semaphore_stats(int64_t* out3) {
  std::lock_guard<std::mutex> lk(g_sem_mu);
  out3[0] = g_sem_permits; out3[1] = g_sem_in_use; out3[2] = g_sem_waits;
  return B2_OK;
}

struct Event { cudaEvent_t ev; };
int b2_event_create(b2_handle* out) {
  B2_TRY
  stream();
  Event* e = new Event();
  CUDA_CHECK(cudaEventCreate(&e->ev));
  *out = to_handle(e);
  B2_CATCH
}
int b2_event_record(b2_handle h) {
  B2_TRY
  CUDA_CHECK(cudaEventRecord(reinterpret_cast<Event*>((intptr_t)h)->ev, stream()));
  B2_CATCH
}
int b2_event_elapsed_ms(b2_handle a, b2_handle b, float* ms) {
  B2_TRY
  Event* ea = reinterpret_cast<Event*>((intptr_t)a);
  Event* eb = reinterpret_cast<Event*>((intptr_t)b);
  CUDA_CHECK(cudaEventSynchronize(eb->ev));
  CUDA_CHECK(cudaEventElapsedTime(ms, ea->ev, eb->ev));
  B2_CATCH
}
int b2_event_close(b2_handle h) {
  B2_TRY
  Event* e = reinterpret_cast<Event*>((intptr_t)h);
  cudaEventDestroy(e->ev);
  delete e;
  B2_CATCH
}

}  // extern "C"
