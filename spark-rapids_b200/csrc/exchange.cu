// exchange.cu — (e): the shuffle exchange over NVLink / NVSwitch.
// Replaces the reference's RapidsShuffleManager data path (GpuShuffleExchangeExecBase.scala:384-536 prepareBatchShuffle-
// Dependency: partition -> contiguousSplit -> serializer; GpuPartitioning.scala:66-99 sliceInternalOnGpuAndClose;
// RapidsShuffleInternalManagerBase.scala:1618 RapidsCachingWriter, :1978 getReaderImpl; the UCX transport in
// shuffle-plugin/): the reference copies each partitioned batch D2H, serialises it on CPU threads and moves it through
// disk/netty or UCX bounce buffers.
//
// Two data paths, one protocol:
//
//  FUSED (b2_exchange_hash, fixed-width columns): ONE kernel hashes the key columns (Spark Murmur3, pmod world — the same
//    ids CPU Spark computes), sorts each 4096-row tile by destination in shared memory and STORES the rows straight into
//    the destination GPU's receive arena through NVLink peer mappings (cudaIpc handles over cudaMalloc'd symmetric
//    arenas, one region per (src, dst) pair, ranges reserved with one atomic per tile and destination).  No partitioned
//    copy of the table is ever written locally, no NCCL send/recv, no host round trip before the data moves.  One
//    ncclAllGather of a 400-byte header per rank (row counts, schema, nullability, has-data flag) is both the size
//    exchange and the completion barrier of the stores (a finished kernel's writes are visible system-wide); ONE
//    device->host read of the gathered headers sizes the output; the receiver copies its W regions out of the arena.
//    Arenas are double buffered by call parity; the header all-gather of call k+1 orders every reader of parity k before
//    any writer of call k+2 (see the ordering argument at b2_exchange_hash).
//
//  NCCL (b2_exchange, any schema incl. strings): table already partitioned by hash.cu; size matrix all-gather, one grouped
//    ncclSend/ncclRecv of every column slice.  Validity travels only for columns that carry NULLs on some rank.
//
// Both take part in the "has data" protocol of GpuShuffleExchangeExec (exec.cu): every rank keeps calling until no rank
// has data left, so ranks with different batch counts (or none) cannot strand their peers inside a collective.
//
// NCCL is bound at run time (dlopen libnccl.so.2) so that the process shares the NCCL that torch.distributed already
// loaded; rendezvous (the 128-byte unique id) is the caller's job.
#include <dlfcn.h>
#include <nccl.h>
#include <algorithm>
#include <mutex>
#include "pack16.cuh"
#include "prim.cuh"
#include "rowops.cuh"
#include "murmur.cuh"

namespace b2 {

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
  const char* (*GetErrorString)(ncclResult_t);
};
static NcclApi g_nccl;
static std::once_flag g_nccl_once;
static bool g_nccl_ok = false;
static std::string g_nccl_err;

static void load_nccl() {
  std::call_once(g_nccl_once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { g_nccl_err = std::string("cannot load libnccl.so.2: ") + dlerror(); return; }
#define B2_SYM(field, name) \
    g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(h, name)); \
    if (!g_nccl.field) { g_nccl_err = std::string("libnccl lacks ") + name; return; }
    B2_SYM(GetUniqueId, "ncclGetUniqueId") B2_SYM(CommInitRank, "ncclCommInitRank") B2_SYM(CommDestroy, "ncclCommDestroy")
    B2_SYM(Send, "ncclSend") B2_SYM(Recv, "ncclRecv") B2_SYM(GroupStart, "ncclGroupStart") B2_SYM(GroupEnd, "ncclGroupEnd")
    B2_SYM(AllGather, "ncclAllGather") B2_SYM(Broadcast, "ncclBroadcast") B2_SYM(GetErrorString, "ncclGetErrorString")
#undef B2_SYM
    g_nccl_ok = true;
  });
  if (!g_nccl_ok) throw Error(B2_ERR_UNSUPPORTED, g_nccl_err);
}
static void nccl_check(ncclResult_t r, const char* what) {
  if (r != ncclSuccess) throw Error(B2_ERR_CUDA, std::string(what) + ": " + g_nccl.GetErrorString(r));
}
#define NCCL_CHECK(x) nccl_check((x), #x)
// an NCCL collective or group that b2_kernel_launch_count counts as one launch (it enqueues one NCCL kernel)
#define NCCL_LAUNCH(x) do { NCCL_CHECK(x); count_launch(); } while (0)

constexpr int XMAX_W = 16;      // ranks of one NVSwitch domain
constexpr int XMAX_COLS = 32;   // columns of an exchanged table on the fused path

// one per rank, all-gathered on every exchange call: sizes, schema and the has-data flag in one fixed-size record
struct XHeader {
  unsigned long long counts[XMAX_W];   // rows this rank stored for each destination (written by the scatter kernel)
  int32_t has_data;                    // this call carries a batch of mine (GpuShuffleExchangeExec termination protocol)
  int32_t ncols;                       // 0 = this rank has not seen a batch yet (adopts the schema of a rank that has)
  int32_t dtype[XMAX_COLS], scale[XMAX_COLS];
  uint32_t nullable_mask;              // bit c: column c carries validity bytes in my regions
  int32_t more;                        // this rank has (or may have) a batch for the NEXT call too: nobody has -> the exchange is over after this call
};

struct Comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  // symmetric receive arenas (fused path)
  bool arena_tried = false, arena_ok = false;
  int next_more = -1;      // b2_comm_set_more: the `more` flag of the next exchange call (-1 = not told: more = has_data, the old protocol)
  int last_any_more = 1;   // max of `more` over the ranks in the last exchange call
  size_t arena_bytes = 0;
  char* arena_local[2] = {nullptr, nullptr};
  char* arena_peer[2][XMAX_W];
  uint64_t epoch = 0;
  XHeader* d_hdr = nullptr;   // my header (device)
  XHeader* d_all = nullptr;   // gathered headers (device)
  XHeader* h_all = nullptr;   // gathered headers (pinned host)
  int64_t bytes_sent = 0, bytes_received = 0, calls = 0;   // payload accounting (bench: exchange GB/s)
  std::vector<int> schema_dtype, schema_scale;               // of the last batch seen (empty tables of exhausted ranks)
};
struct TableRefLite { Table* t = nullptr; ~TableRefLite() { if (t) table_release(t); } };
static Comm* comm_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null communicator handle");
  return reinterpret_cast<Comm*>((intptr_t)h);
}

// ---- symmetric arenas -------------------------------------------------------------------------------------------------------
static void arena_release(Comm* c, bool barrier) {   // barrier: a collective decision of the caller (same on every rank)
  for (int p = 0; p < 2; p++)
    for (int r = 0; r < c->world; r++) {
      if (r != c->rank && c->arena_peer[p][r]) cudaIpcCloseMemHandle(c->arena_peer[p][r]);
      c->arena_peer[p][r] = nullptr;
    }
  if (barrier) {   // nobody frees an arena a peer still has mapped
    DevBuf a(8), b(8 * (size_t)c->world);
    NCCL_CHECK(g_nccl.AllGather(a.p, b.p, 8, ncclInt8, c->comm, stream()));
    CUDA_CHECK(cudaStreamSynchronize(stream()));
  }
  for (int p = 0; p < 2; p++)
    if (c->arena_local[p]) { cudaFree(c->arena_local[p]); c->arena_local[p] = nullptr; }
  c->arena_ok = false; c->arena_bytes = 0;
}

// collective: every rank allocates two arenas of `bytes` and maps every peer's arenas (cudaIpc over NVLink P2P)
static bool arena_setup(Comm* c, size_t bytes) {
  cudaStream_t s = stream();
  CUDA_CHECK(cudaStreamSynchronize(s));
  arena_release(c, c->arena_ok);   // arena_ok is the same on every rank
  const int W = c->world;
  bool ok = true;
  for (int p = 0; p < 2 && ok; p++)
    if (cudaMalloc((void**)&c->arena_local[p], bytes) != cudaSuccess) { cudaGetLastError(); ok = false; }
  struct Rec { cudaIpcMemHandle_t h[2]; int32_t ok; int32_t pad; };
  Rec mine; memset(&mine, 0, sizeof(mine));
  mine.ok = ok ? 1 : 0;
  for (int p = 0; p < 2 && ok; p++)
    if (cudaIpcGetMemHandle(&mine.h[p], c->arena_local[p]) != cudaSuccess) { cudaGetLastError(); mine.ok = 0; ok = false; }
  DevBuf d_mine(sizeof(Rec)), d_all(sizeof(Rec) * W);
  CUDA_CHECK(cudaMemcpyAsync(d_mine.p, &mine, sizeof(Rec), cudaMemcpyHostToDevice, s));
  NCCL_CHECK(g_nccl.AllGather(d_mine.p, d_all.p, sizeof(Rec), ncclInt8, c->comm, s));
  std::vector<Rec> all(W);
  CUDA_CHECK(cudaMemcpyAsync(all.data(), d_all.p, sizeof(Rec) * W, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  bool everyone = true;
  for (int r = 0; r < W; r++) everyone = everyone && all[r].ok;
  int32_t mapped = everyone ? 1 : 0;
  if (everyone) {
    for (int p = 0; p < 2; p++)
      for (int r = 0; r < W; r++) {
        if (r == c->rank) { c->arena_peer[p][r] = c->arena_local[p]; continue; }
        void* ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[r].h[p], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); mapped = 0; ptr = nullptr; }
        c->arena_peer[p][r] = (char*)ptr;
      }
  }
  // second round: the fused path is used only when EVERY rank mapped every peer (the decision must be collective)
  DevBuf d_m(4), d_ma(4 * (size_t)W);
  CUDA_CHECK(cudaMemcpyAsync(d_m.p, &mapped, 4, cudaMemcpyHostToDevice, s));
  NCCL_CHECK(g_nccl.AllGather(d_m.p, d_ma.p, 4, ncclInt8, c->comm, s));
  std::vector<int32_t> ma(W);
  CUDA_CHECK(cudaMemcpyAsync(ma.data(), d_ma.p, 4 * (size_t)W, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  bool all_mapped = true;
  for (int r = 0; r < W; r++) all_mapped = all_mapped && ma[r];
  if (!all_mapped) { arena_release(c, true); return false; }
  c->arena_bytes = bytes; c->arena_ok = true;
  return true;
}

// ---- fused hash-partition -> peer-store kernel -------------------------------------------------------------------------------
constexpr int XS_NT = 256, XS_STEPS = 16, XS_TILE = XS_NT * XS_STEPS;   // 4096 rows per tile
struct XPlan {
  int32_t W, me, ncols, single;   // single: SinglePartition (everything to rank 0)
  int64_t cap;                    // rows a (src, dst) region holds
  int64_t region_bytes;           // bytes of one src region inside a dst arena
  char* arena[XMAX_W];            // destination arenas of this call's parity (peer mappings)
  int32_t width[XMAX_COLS];
  int64_t col_off[XMAX_COLS];     // byte offset of column c inside a region
  int64_t val_off[XMAX_COLS];     // byte offset of its validity bytes inside a region
  const void* in[XMAX_COLS];
  const uint32_t* in_valid[XMAX_COLS];   // null = this column ships no validity
  const int32_t* sel;                    // selection vector (row ids into the batch) or null: late materialisation of a filter below
};

// per-tile geometry of the destination runs (shared memory): stage rows [start, start_next) belong to destination p in
// destination order; rows [start, end) fit the (me -> p) region; destination row = stage row + c
struct XRuns {
  int start[XMAX_W + 1];
  int end[XMAX_W];
  long long c[XMAX_W];
};

// one column of one tile: the values are scattered into destination order in shared memory, then every destination's run is
// streamed out.  Every store that can be is a 16-byte store to a 16-byte aligned address of the destination region (512
// contiguous bytes per warp store, the shape NVLink carries at full rate): the run is cut at the destination's vector
// boundaries, a vector reads its V (in general unaligned) elements from shared memory, and only the < V rows in front of the
// first and behind the last whole vector leave one by one.  Rows past the region's capacity are dropped here and counted by
// the caller (grow + retry).  VALID: the source is a validity bit mask, shipped as one byte per row.
template <typename T, bool VALID>
__device__ __forceinline__ void xs_move_column(const XPlan& pl, int64_t off_bytes, const void* __restrict__ in, T* stage, const uint16_t* lpos,
                                               int64_t tile_base, int64_t n, const XRuns& rn) {
  // loads in explicit batches: all of a batch's (dependent: selection vector -> value) loads are in flight before the first
  // shared-memory store waits for one.  (Left to the compiler under a register cap, the 16 fully unrolled steps became 16
  // serial load -> store round trips: ncu put 60 % of the kernel's stall samples on the STS / first use of the loaded value.)
  // The batch loop itself is NOT unrolled and the stage positions live in shared memory, which keeps the kernel small enough
  // to hold a batch in registers without spilling.
  constexpr int XB = sizeof(T) >= 16 ? 4 : 8;
#pragma unroll 1
  for (int j0 = 0; j0 < XS_STEPS; j0 += XB) {
    int64_t src[XB];
    T v[XB];
#pragma unroll
    for (int b = 0; b < XB; b++) {
      const int64_t i = tile_base + (int64_t)(j0 + b) * XS_NT + threadIdx.x;
      src[b] = i < n ? (pl.sel ? (int64_t)pl.sel[i] : i) : -1;
    }
#pragma unroll
    for (int b = 0; b < XB; b++) {
      if (src[b] >= 0) {
        if constexpr (VALID) v[b] = (T)bit_get(reinterpret_cast<const uint32_t*>(in), src[b]);
        else v[b] = reinterpret_cast<const T*>(in)[src[b]];
      }
    }
#pragma unroll
    for (int b = 0; b < XB; b++) if (src[b] >= 0) stage[lpos[(j0 + b) * XS_NT + threadIdx.x]] = v[b];
  }
  __syncthreads();
  constexpr int V = sizeof(T) >= 16 ? 1 : 16 / (int)sizeof(T);
  for (int p = 0; p < pl.W; p++) {
    const int st = rn.start[p], en = rn.end[p];
    if (en <= st) continue;
    const long long c = rn.c[p];
    T* out = reinterpret_cast<T*>(pl.arena[p] + (int64_t)pl.me * pl.region_bytes + off_bytes) + c;   // out[k] = destination of stage row k
    if (V == 1) { for (int k = st + threadIdx.x; k < en; k += XS_NT) out[k] = stage[k]; continue; }
    const int head = min(en - st, (V - (int)((st + c) & (V - 1))) & (V - 1));
    const int vlo = st + head;
    const int nvec = (en - vlo) / V;
#pragma unroll 4
    for (int v = threadIdx.x; v < nvec; v += XS_NT) {   // independent iterations: up to four vectors in flight per thread
      const int kk = vlo + v * V;
      *reinterpret_cast<uint4*>(out + kk) = pack16<T>(stage + kk);
    }
    const int vhi = vlo + nvec * V;
    const int nb = head + (en - vhi);   // < 2 V <= 32 rows
    if ((int)threadIdx.x < nb) { const int k = (int)threadIdx.x < head ? st + threadIdx.x : vhi + ((int)threadIdx.x - head); out[k] = stage[k]; }
  }
  __syncthreads();
}

// KM: how a row's destination is computed.  0 = generic (any key columns, NULLs), 1 = ONE 64-bit integer-like key column without
// NULLs (INT64 / TIMESTAMP / DECIMAL64: Spark hashes the raw long), 2 = ONE INT32 / DATE32 column without NULLs.
template <int KM>
__global__ void __launch_bounds__(XS_NT, 3) xchg_scatter_kernel(const __grid_constant__ KeyCols keys, const __grid_constant__ XPlan pl, int64_t n, uint32_t seed,
                                                             unsigned long long* __restrict__ counters) {
  extern __shared__ __align__(16) char stage_raw[];   // XS_TILE * widest column
  __shared__ int s_wcnt[XS_NT / 32][XMAX_W];          // rows of (warp, destination); then the warp's offset inside the destination's run
  __shared__ int s_cnt[XMAX_W];
  __shared__ long long s_gbase[XMAX_W];
  __shared__ uint16_t s_lpos[XS_TILE];   // rank among the warp's rows for the destination, then the stage position
  __shared__ uint8_t s_pid[XS_TILE];
  __shared__ XRuns rn;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  const int64_t ntiles = (n + XS_TILE - 1) / XS_TILE;
  const bool pow2 = (pl.W & (pl.W - 1)) == 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t tile_base = tile * XS_TILE;
    for (int k = threadIdx.x; k < (XS_NT / 32) * XMAX_W; k += XS_NT) (&s_wcnt[0][0])[k] = 0;
    __syncthreads();
    // destination of every row (Spark Murmur3 over the key columns, pmod world) and its rank among the warp's rows for that
    // destination: one match_any per 32 rows, running counts per (warp, destination) — no atomics, deterministic order.
    // Batches of XH rows per thread: XH selection-vector loads, then XH key loads in flight at once.
    constexpr int XH = 8;
#pragma unroll 1
    for (int j0 = 0; j0 < XS_STEPS; j0 += XH) {
      int64_t src[XH];
      uint32_t h[XH];
#pragma unroll
      for (int b = 0; b < XH; b++) {
        const int64_t i = tile_base + (int64_t)(j0 + b) * XS_NT + threadIdx.x;
        src[b] = i < n ? (pl.sel ? (int64_t)pl.sel[i] : i) : -1;
      }
      if (KM == 1) {
        uint64_t kv[XH];
#pragma unroll
        for (int b = 0; b < XH; b++) kv[b] = src[b] >= 0 ? reinterpret_cast<const uint64_t*>(keys.c[0].data)[src[b]] : 0ull;
#pragma unroll
        for (int b = 0; b < XH; b++) h[b] = hash_long(kv[b], seed);
      } else if (KM == 2) {
        uint32_t kv[XH];
#pragma unroll
        for (int b = 0; b < XH; b++) kv[b] = src[b] >= 0 ? reinterpret_cast<const uint32_t*>(keys.c[0].data)[src[b]] : 0u;
#pragma unroll
        for (int b = 0; b < XH; b++) h[b] = hash_int(kv[b], seed);
      } else {
#pragma unroll
        for (int b = 0; b < XH; b++) {
          h[b] = seed;
          if (src[b] >= 0 && !pl.single) for (int c = 0; c < keys.n; c++) h[b] = murmur_col(keys.c[c], src[b], h[b]);
        }
      }
#pragma unroll
      for (int b = 0; b < XH; b++) {
        int p = -1;
        if (src[b] >= 0) {
          if (pl.single) p = 0;
          else if (pow2) p = (int)(h[b] & (uint32_t)(pl.W - 1));   // pmod of a two's complement int by a power of two
          else { int32_t v = (int32_t)h[b] % pl.W; if (v < 0) v += pl.W; p = v; }
        }
        const uint32_t m = __match_any_sync(0xffffffffu, p);
        const int leader = __ffs(m) - 1;
        int first = 0;
        if (p >= 0 && lane == leader) { first = s_wcnt[warp][p]; s_wcnt[warp][p] = first + __popc(m); }
        first = __shfl_sync(0xffffffffu, first, leader);
        __syncwarp();
        const int li = (j0 + b) * XS_NT + threadIdx.x;
        s_pid[li] = (uint8_t)p;
        s_lpos[li] = (uint16_t)(first + __popc(m & lt));
      }
    }
    __syncthreads();
    if (threadIdx.x < pl.W) {   // offsets of the warps inside the destination's run; one reservation per tile and destination
      const int p = threadIdx.x;
      int run = 0;
#pragma unroll
      for (int w = 0; w < XS_NT / 32; w++) { const int c = s_wcnt[w][p]; s_wcnt[w][p] = run; run += c; }
      s_cnt[p] = run;
      s_gbase[p] = run ? (long long)atomicAdd(&counters[p], (unsigned long long)run) : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int run = 0;
      for (int p = 0; p < pl.W; p++) {
        const long long room = pl.cap - s_gbase[p];
        rn.start[p] = run;
        rn.end[p] = run + (int)max(0LL, min(room, (long long)s_cnt[p]));
        rn.c[p] = s_gbase[p] - run;
        run += s_cnt[p];
      }
      rn.start[pl.W] = run;
    }
    __syncthreads();
    for (int li = threadIdx.x; li < XS_TILE; li += XS_NT) {   // same thread as above: no barrier needed for its own entries
      const int p = s_pid[li];
      if (p != 0xff) s_lpos[li] = (uint16_t)(rn.start[p] + s_wcnt[warp][p] + s_lpos[li]);
    }
    for (int c = 0; c < pl.ncols; c++) {
      switch (pl.width[c]) {
        case 1: xs_move_column<uint8_t, false>(pl, pl.col_off[c], pl.in[c], (uint8_t*)stage_raw, s_lpos, tile_base, n, rn); break;
        case 2: xs_move_column<uint16_t, false>(pl, pl.col_off[c], pl.in[c], (uint16_t*)stage_raw, s_lpos, tile_base, n, rn); break;
        case 4: xs_move_column<uint32_t, false>(pl, pl.col_off[c], pl.in[c], (uint32_t*)stage_raw, s_lpos, tile_base, n, rn); break;
        case 8: xs_move_column<uint64_t, false>(pl, pl.col_off[c], pl.in[c], (uint64_t*)stage_raw, s_lpos, tile_base, n, rn); break;
        default: xs_move_column<uint4, false>(pl, pl.col_off[c], pl.in[c], (uint4*)stage_raw, s_lpos, tile_base, n, rn); break;
      }
      // validity as one byte per row (only for columns that carry NULLs here)
      if (pl.in_valid[c]) xs_move_column<uint8_t, true>(pl, pl.val_off[c], pl.in_valid[c], (uint8_t*)stage_raw, s_lpos, tile_base, n, rn);
    }
  }
}

// receiver side: all (source region, column) segments of one exchange call copied out of the arena by ONE kernel
// (W x ncols cudaMemcpyAsync calls would cost more in launch latency than in bytes at W = 8)
struct CopySeg { const char* src; char* dst; int64_t bytes; };
__global__ void xchg_copy_out_kernel(const CopySeg* __restrict__ segs, int nsegs) {
  for (int sgi = blockIdx.y; sgi < nsegs; sgi += gridDim.y) {
    const CopySeg sg = segs[sgi];
    const uintptr_t a = (uintptr_t)sg.src | (uintptr_t)sg.dst | (uintptr_t)sg.bytes;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, step = (int64_t)gridDim.x * blockDim.x;
    if ((a & 15) == 0) { for (int64_t i = t0; i < sg.bytes / 16; i += step) reinterpret_cast<uint4*>(sg.dst)[i] = reinterpret_cast<const uint4*>(sg.src)[i]; }
    else if ((a & 7) == 0) { for (int64_t i = t0; i < sg.bytes / 8; i += step) reinterpret_cast<uint64_t*>(sg.dst)[i] = reinterpret_cast<const uint64_t*>(sg.src)[i]; }
    else if ((a & 3) == 0) { for (int64_t i = t0; i < sg.bytes / 4; i += step) reinterpret_cast<uint32_t*>(sg.dst)[i] = reinterpret_cast<const uint32_t*>(sg.src)[i]; }
    else { for (int64_t i = t0; i < sg.bytes; i += step) sg.dst[i] = sg.src[i]; }
  }
}

// receiver side: validity bytes of one source region -> bits at an arbitrary row offset of the output mask (pre-zeroed)
__global__ void bytes_to_bits_at_kernel(const uint8_t* __restrict__ in, int64_t n, uint32_t* __restrict__ bits, int64_t start) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (in == nullptr || in[i]) atomicOr(&bits[(start + i) >> 5], 1u << ((start + i) & 31));
}

__global__ void bits_to_bytes_kernel(const uint32_t* __restrict__ bits, int64_t n, uint8_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = bits ? (uint8_t)bit_get(bits, i) : 1;
}
__global__ void bytes_to_bits_kernel(const uint8_t* __restrict__ in, int64_t n, uint32_t* __restrict__ bits) {
  const int64_t nround = (n + 31) & ~(int64_t)31;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
    const bool v = i < n && in[i] != 0;
    const uint32_t b = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && i < n) bits[i >> 5] = b;
  }
}
__global__ void lengths_kernel(const int32_t* __restrict__ offsets, int64_t n, int32_t* __restrict__ len) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) len[i] = offsets[i + 1] - offsets[i];
}

// layout of one (src -> dst) region for a schema: identical on every rank (depends on widths and the arena size only)
struct XLayout { int64_t cap, region_bytes; int64_t col_off[XMAX_COLS], val_off[XMAX_COLS]; };
static XLayout region_layout(size_t arena_bytes, int W, const std::vector<int>& widths) {
  XLayout L; memset(&L, 0, sizeof(L));
  L.region_bytes = (int64_t)((arena_bytes / (size_t)W) & ~(size_t)255);
  int64_t row_bytes = 0;
  for (int w : widths) row_bytes += w + 1;
  const int64_t slack = 512 * (int64_t)widths.size();
  L.cap = row_bytes ? (L.region_bytes - slack) / row_bytes : 0;
  if (L.cap < 0) L.cap = 0;
  L.cap &= ~(int64_t)63;
  int64_t off = 0;
  for (size_t c = 0; c < widths.size(); c++) {
    L.col_off[c] = off; off = (off + L.cap * widths[c] + 255) & ~(int64_t)255;
    L.val_off[c] = off; off = (off + L.cap + 255) & ~(int64_t)255;
  }
  return L;
}

static Table* empty_table_of(const std::vector<int>& dtypes, const std::vector<int>& scales) {
  ColsGuard outs;
  for (size_t i = 0; i < dtypes.size(); i++) {
    if (dtypes[i] == B2_STRING) {
      std::unique_ptr<Column> c(new Column());
      c->dtype = B2_STRING; c->size = 0; c->offsets = DevBuf(4); c->data = DevBuf(0);
      CUDA_CHECK(cudaMemsetAsync(c->offsets.p, 0, 4, stream()));
      outs.v.push_back(c.release());
    } else outs.v.push_back(new_column(dtypes[i], scales[i], 0, false));
  }
  return new_table(outs.release());
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_comm_unique_id(uint8_t* out128) {
  B2_TRY
  load_nccl();
  ncclUniqueId id;
  NCCL_CHECK(g_nccl.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  memcpy(out128, &id, 128);
  B2_CATCH
}

int b2_comm_init(const uint8_t* id128, int32_t rank, int32_t world, b2_handle* out_comm) {
  B2_TRY
  load_nccl();
  stream();  // binds the device
  B2_CHECK(world >= 1 && world <= XMAX_W && rank >= 0 && rank < world, "communicator of 1..16 ranks");
  std::unique_ptr<Comm> c(new Comm());
  c->rank = rank; c->world = world;
  memset(c->arena_peer, 0, sizeof(c->arena_peer));
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  NCCL_CHECK(g_nccl.CommInitRank(&c->comm, world, id, rank));
  CUDA_CHECK(cudaMalloc((void**)&c->d_hdr, sizeof(XHeader)));
  CUDA_CHECK(cudaMalloc((void**)&c->d_all, sizeof(XHeader) * world));
  CUDA_CHECK(cudaHostAlloc((void**)&c->h_all, sizeof(XHeader) * world, cudaHostAllocDefault));
  *out_comm = to_handle(c.release());
  B2_CATCH
}

int b2_comm_close(b2_handle h) {
  B2_TRY
  Comm* c = comm_from(h);
  cudaStreamSynchronize(stream());
  arena_release(c, false);
  if (c->d_hdr) cudaFree(c->d_hdr);
  if (c->d_all) cudaFree(c->d_all);
  if (c->h_all) cudaFreeHost(c->h_all);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  delete c;
  B2_CATCH
}

// collective: map the peer arenas if that has not been tried yet; *ok = the fused path is usable on EVERY rank
int b2_comm_fused_ready(b2_handle h, int32_t* ok) {
  B2_TRY
  Comm* c = comm_from(h);
  if (!c->arena_tried) {
    c->arena_tried = true;
    size_t mb = 1024;
    if (const char* e = getenv("B2_EXCHANGE_ARENA_MB")) mb = (size_t)std::max(1, atoi(e));
    if (!getenv("B2_EXCHANGE_NO_FUSED")) arena_setup(c, mb << 20);   // a world of one stores into its own arena (probe / single-GPU plans)
  }
  *ok = c->arena_ok ? 1 : 0;
  B2_CATCH
}

// collective max of one int per rank (plan-level agreements of the exec layer, e.g. "does any rank's batch carry strings")
int b2_comm_allmax(b2_handle h, int32_t value, int32_t* out) {
  B2_TRY
  Comm* c = comm_from(h);
  cudaStream_t s = stream();
  DevBuf a(4), b(4 * (size_t)c->world);
  h2d_bytes(a.p, &value, 4);
  NCCL_LAUNCH(g_nccl.AllGather(a.p, b.p, 4, ncclInt8, c->comm, s));
  std::vector<int32_t> all(c->world);
  CUDA_CHECK(cudaMemcpyAsync(all.data(), b.p, 4 * (size_t)c->world, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  int32_t m = all[0];
  for (int v : all) m = std::max(m, v);
  *out = m;
  B2_CATCH
}

// Termination without an extra (empty) round: a caller that looks one batch ahead tells the next exchange call whether it
// will come again with data; after the call b2_comm_any_more says whether ANY rank will.  Without b2_comm_set_more the flag
// defaults to "this call carried data", i.e. the exchange ends with the first call in which nobody had a batch.
int b2_comm_set_more(b2_handle h, int32_t more) {
  B2_TRY
  comm_from(h)->next_more = more ? 1 : 0;
  B2_CATCH
}
int b2_comm_any_more(b2_handle h, int32_t* out) {
  B2_TRY
  *out = comm_from(h)->last_any_more;
  B2_CATCH
}

int b2_comm_stats(b2_handle h, int64_t* out4) {
  B2_TRY
  Comm* c = comm_from(h);
  out4[0] = c->bytes_sent; out4[1] = c->bytes_received; out4[2] = c->calls; out4[3] = c->arena_ok ? (int64_t)c->arena_bytes : 0;
  B2_CATCH
}

// Fused GpuHashPartitioning + shuffle write + shuffle read.  `table` = 0: this rank has no batch for this call (its child
// is exhausted); it still takes part.  *any_data = some rank carried a batch; when 0 the exchange is over on every rank and
// *out_table is 0.
//
// Arena reuse is safe without an extra barrier: call k stores into parity k&1.  A reader copies its regions out on its
// stream BEFORE it enqueues the header all-gather of call k+1; a writer of call k+2 (same parity) launches its scatter
// only AFTER its own all-gather of call k+1 returned data from every rank, i.e. after every reader's stream passed its
// copy-out of call k.
int b2_exchange_hash(b2_handle comm, b2_handle table, const int32_t* key_cols, int32_t nkeys, int32_t seed,
                     b2_handle* out_table, int32_t* any_data) {
  return b2_exchange_hash_sel(comm, table, 0, nullptr, 0, key_cols, nkeys, seed, out_table, any_data);
}

// key_cols index the columns of `table` (the unpruned batch); out_cols (nout > 0) are the columns that travel
int b2_exchange_hash_sel(b2_handle comm, b2_handle table, b2_handle selection, const int32_t* out_cols, int32_t nout,
                         const int32_t* key_cols, int32_t nkeys, int32_t seed, b2_handle* out_table, int32_t* any_data) {
  B2_TRY
  Comm* c = comm_from(comm);
  const int W = c->world, me = c->rank;
  Table* full = table ? table_from(table) : nullptr;
  // the travelling columns as a (non-owning) view; keys are read from the full batch
  Table view;
  struct Unhook { Table& t; ~Unhook() { t.cols.clear(); } } unhook{view};
  Table* t = full;
  if (full && nout > 0) {
    for (int i = 0; i < nout; i++) {
      B2_CHECK(out_cols[i] >= 0 && out_cols[i] < (int)full->cols.size(), "exchange: output column out of range");
      view.cols.push_back(full->cols[out_cols[i]]);
    }
    view.rows = full->rows;
    t = &view;
  }
  const int32_t* sel = nullptr;
  int64_t nsend = t ? t->rows : 0;
  if (selection) {
    Column* sc = col_from(selection);
    B2_CHECK(sc->dtype == B2_INT32 && full, "selection vector must be INT32 over a batch");
    sel = sc->data.as<int32_t>(); nsend = sc->size;
  }
  cudaStream_t s = stream();
  *out_table = 0; *any_data = 0;
  if (t) {
    B2_CHECK((int)t->cols.size() >= 1 && (int)t->cols.size() <= XMAX_COLS, "fused exchange: 1..32 columns");
    for (auto* col : t->cols) if (col->dtype == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "fused exchange: STRING columns take the NCCL path (b2_exchange)");
  }
  // the schema travels in the header of every rank that has a batch; a rank without one adopts it from a peer (a communicator
  // serves many exchange nodes with different schemas, so nothing is remembered between calls)
  c->schema_dtype.clear(); c->schema_scale.clear();
  if (t) for (auto* col : t->cols) { c->schema_dtype.push_back(col->dtype); c->schema_scale.push_back(col->scale); }
  { int32_t ok = 0; int rc = b2_comm_fused_ready(comm, &ok); if (rc != B2_OK) return rc; }
  if (!c->arena_ok) throw Error(B2_ERR_UNSUPPORTED, "fused exchange: peer arenas could not be mapped (no NVLink P2P / IPC between the ranks)");
  KeyCols keys; memset(&keys, 0, sizeof(keys));
  if (full && nkeys > 0) keys = key_cols_of(full, key_cols, nkeys);
  XHeader hdr; memset(&hdr, 0, sizeof(hdr));
  hdr.has_data = t ? 1 : 0;
  hdr.more = c->next_more >= 0 ? c->next_more : hdr.has_data; c->next_more = -1;
  hdr.ncols = (int)c->schema_dtype.size();
  for (int i = 0; i < hdr.ncols; i++) { hdr.dtype[i] = c->schema_dtype[i]; hdr.scale[i] = c->schema_scale[i]; }
  if (t) for (int i = 0; i < hdr.ncols; i++) if (t->cols[i]->nullable()) hdr.nullable_mask |= 1u << i;
  std::vector<int> widths;
  for (int i = 0; i < hdr.ncols; i++) widths.push_back(dtype_width(hdr.dtype[i]));
  std::vector<XHeader> all(W);
  XLayout L;
  for (int attempt = 0;; attempt++) {
    const int parity = (int)(c->epoch & 1);
    c->epoch++;
    L = region_layout(c->arena_bytes, W, widths);
    h2d_bytes(c->d_hdr, &hdr, sizeof(hdr));
    if (t && nsend > 0) {
      XPlan pl; memset(&pl, 0, sizeof(pl));
      pl.sel = sel;
      pl.W = W; pl.me = me; pl.ncols = hdr.ncols; pl.single = nkeys == 0 ? 1 : 0;
      pl.cap = L.cap; pl.region_bytes = L.region_bytes;
      for (int r = 0; r < W; r++) pl.arena[r] = c->arena_peer[parity][r];
      int maxw = 1;
      for (int i = 0; i < hdr.ncols; i++) {
        pl.width[i] = widths[i]; pl.col_off[i] = L.col_off[i]; pl.val_off[i] = L.val_off[i];
        pl.in[i] = t->cols[i]->data.p; pl.in_valid[i] = t->cols[i]->validity();
        maxw = std::max(maxw, widths[i]);
      }
      const int smem = XS_TILE * maxw;
      // key mode: one integer key column without NULLs (every TPC-H join key) skips the generic per-row type dispatch
      int km = 0;
      if (keys.n == 1 && !keys.c[0].valid) {
        const int dt = keys.c[0].dtype;
        if (dt == B2_INT64 || dt == B2_TIMESTAMP_US || dt == B2_DECIMAL64) km = 1;
        else if (dt == B2_INT32 || dt == B2_DATE32) km = 2;
      }
      auto kern = km == 1 ? xchg_scatter_kernel<1> : (km == 2 ? xchg_scatter_kernel<2> : xchg_scatter_kernel<0>);
      const int64_t ntiles = (nsend + XS_TILE - 1) / XS_TILE;
      const int per_sm = std::max(1, std::min(3, (200 * 1024) / (smem + 2048)));
      const int grid = (int)std::min<int64_t>(ntiles, (int64_t)sm_count() * per_sm);
      launch("xchg_scatter_kernel", kern, grid, XS_NT, smem, s, keys, pl, nsend, (uint32_t)seed, c->d_hdr->counts);
    }
    {
      // sizes + schema + has-data of every rank; also the completion barrier of every rank's peer stores
      KernelTimer kt("xchg_header_allgather");
      NCCL_LAUNCH(g_nccl.AllGather(c->d_hdr, c->d_all, sizeof(XHeader), ncclInt8, c->comm, s));
    }
    CUDA_CHECK(cudaMemcpyAsync(c->h_all, c->d_all, sizeof(XHeader) * W, cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    memcpy(all.data(), c->h_all, sizeof(XHeader) * W);
    // a rank without a schema adopts one (it may receive rows); every rank sees the same headers
    int src_schema = -1;
    for (int r = 0; r < W; r++) if (all[r].ncols > 0) { src_schema = r; break; }
    if (hdr.ncols == 0 && src_schema >= 0) {
      hdr.ncols = all[src_schema].ncols;
      c->schema_dtype.assign(all[src_schema].dtype, all[src_schema].dtype + hdr.ncols);
      c->schema_scale.assign(all[src_schema].scale, all[src_schema].scale + hdr.ncols);
      for (int i = 0; i < hdr.ncols; i++) { hdr.dtype[i] = c->schema_dtype[i]; hdr.scale[i] = c->schema_scale[i]; }
      widths.clear();
      for (int i = 0; i < hdr.ncols; i++) widths.push_back(dtype_width(hdr.dtype[i]));
      L = region_layout(c->arena_bytes, W, widths);
    }
    for (int r = 0; r < W; r++) {
      if (all[r].ncols == 0) continue;
      B2_CHECK(all[r].ncols == hdr.ncols, "exchange: ranks disagree on the number of columns");
      for (int i = 0; i < hdr.ncols; i++) B2_CHECK(all[r].dtype[i] == hdr.dtype[i], "exchange: ranks disagree on a column type");
    }
    unsigned long long worst = 0;
    for (int r = 0; r < W; r++) for (int d = 0; d < W; d++) worst = std::max(worst, all[r].counts[d]);
    if ((int64_t)worst <= L.cap) break;
    // some (src, dst) stream did not fit its region: every rank sees the same matrix and grows the arenas together
    if (attempt >= 3) throw Error(B2_ERR_OOM, "fused exchange: a partition does not fit the receive arena");
    int64_t row_bytes = 0;
    for (int w : widths) row_bytes += w + 1;
    size_t need = (size_t)((int64_t)worst * row_bytes * W * 5 / 4 + (int64_t)W * 1024 * (int64_t)widths.size() + (1 << 20));
    size_t nb = c->arena_bytes;
    while (nb < need) nb <<= 1;
    if (!arena_setup(c, nb)) throw Error(B2_ERR_OOM, "fused exchange: could not grow the receive arenas");
    c->epoch = 0;
  }
  const int parity = (int)((c->epoch - 1) & 1);
  int anyd = 0;
  for (int r = 0; r < W; r++) anyd |= all[r].has_data;
  c->last_any_more = 0;
  for (int r = 0; r < W; r++) c->last_any_more |= all[r].more;
  *any_data = anyd;
  c->calls++;
  if (!anyd) return B2_OK;
  if (hdr.ncols == 0) throw Error(B2_ERR_INVALID, "exchange: no rank knows the schema");
  int64_t out_rows = 0;
  for (int r = 0; r < W; r++) if (!all[r].has_data) for (int d = 0; d < W; d++) all[r].counts[d] = 0;   // a rank without a batch stored nothing
  for (int r = 0; r < W; r++) out_rows += (int64_t)all[r].counts[me];
  if (out_rows > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "exchange result exceeds 2^31-1 rows");
  uint32_t any_null = 0;
  for (int r = 0; r < W; r++) if (all[r].counts[me]) any_null |= all[r].nullable_mask;
  ColsGuard outs;
  int64_t row_bytes = 0;
  for (int i = 0; i < hdr.ncols; i++) {
    const bool nullable = (any_null >> i) & 1u;
    Column* oc = new_column(hdr.dtype[i], hdr.scale[i], out_rows, nullable);
    outs.v.push_back(oc);
    if (nullable && out_rows) CUDA_CHECK(cudaMemsetAsync(oc->valid.p, 0, oc->valid.bytes, s));
    row_bytes += widths[i];
  }
  {
    KernelTimer kt("xchg_copy_out");
    std::vector<CopySeg> segs;
    int64_t row = 0, biggest = 0;
    for (int r = 0; r < W; r++) {
      const int64_t cnt = (int64_t)all[r].counts[me];
      if (!cnt) continue;
      const char* region = c->arena_local[parity] + (int64_t)r * L.region_bytes;
      for (int i = 0; i < hdr.ncols; i++) {
        Column* oc = outs.v[i];
        segs.push_back({region + L.col_off[i], oc->data.as<char>() + row * widths[i], cnt * widths[i]});
        biggest = std::max(biggest, cnt * widths[i]);
        if (oc->valid.p) {
          const uint8_t* vb = ((all[r].nullable_mask >> i) & 1u) ? reinterpret_cast<const uint8_t*>(region + L.val_off[i]) : nullptr;
          launch(bytes_to_bits_at_kernel, grid_for(cnt, 256), 256, 0, s, vb, cnt, oc->valid.as<uint32_t>(), row);
        }
      }
      row += cnt;
    }
    if (!segs.empty()) {
      DevBuf d_segs(segs.size() * sizeof(CopySeg));
      h2d_bytes(d_segs.p, segs.data(), segs.size() * sizeof(CopySeg));
      const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((biggest / 16 + 255) / 256, (int64_t)sm_count() * 4));
      const int gy = (int)std::min<size_t>(segs.size(), 64);
      launch(xchg_copy_out_kernel, dim3(gx, gy), 256, 0, s, d_segs.as<CopySeg>(), (int)segs.size());
      // d_segs is stream-ordered: freed after the kernel
    }
  }
  if (t) for (int d = 0; d < W; d++) if (d != me) c->bytes_sent += (int64_t)all[me].counts[d] * row_bytes;
  for (int r = 0; r < W; r++) if (r != me) c->bytes_received += (int64_t)all[r].counts[me] * row_bytes;
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

// NCCL path.  `partitioned_table` = 0 / offsets = null: this rank has no batch for this call.
int b2_exchange_ex(b2_handle comm, b2_handle partitioned_table, const int32_t* offsets, b2_handle* out_table, int32_t* any_data) {
  B2_TRY
  Comm* c = comm_from(comm);
  const int W = c->world, me = c->rank;
  cudaStream_t s = stream();
  *out_table = 0; *any_data = 0;
  TableRefLite keep;   // an empty stand-in table for a rank without a batch (schema of its last batch)
  Table* t = partitioned_table ? table_from(partitioned_table) : nullptr;
  std::vector<int32_t> zero_offs(W + 1, 0);
  const bool mine = t != nullptr;
  c->schema_dtype.clear(); c->schema_scale.clear();   // nothing is remembered between calls: see b2_exchange_hash
  if (t) for (auto* col : t->cols) { c->schema_dtype.push_back(col->dtype); c->schema_scale.push_back(col->scale); }
  else offsets = zero_offs.data();
  // round 0: who has data, and the schema for ranks that never saw a batch
  XHeader hdr; memset(&hdr, 0, sizeof(hdr));
  hdr.has_data = mine ? 1 : 0;
  hdr.more = c->next_more >= 0 ? c->next_more : hdr.has_data; c->next_more = -1;
  hdr.ncols = (int)std::min<size_t>(c->schema_dtype.size(), XMAX_COLS);
  B2_CHECK(c->schema_dtype.size() <= (size_t)XMAX_COLS, "exchange: more than 32 columns");
  for (int i = 0; i < hdr.ncols; i++) { hdr.dtype[i] = c->schema_dtype[i]; hdr.scale[i] = c->schema_scale[i]; }
  if (t) for (int i = 0; i < hdr.ncols; i++) if (t->cols[i]->nullable()) hdr.nullable_mask |= 1u << i;
  h2d_bytes(c->d_hdr, &hdr, sizeof(hdr));
  NCCL_LAUNCH(g_nccl.AllGather(c->d_hdr, c->d_all, sizeof(XHeader), ncclInt8, c->comm, s));
  CUDA_CHECK(cudaMemcpyAsync(c->h_all, c->d_all, sizeof(XHeader) * W, cudaMemcpyDeviceToHost, s));
  // char offsets of the string columns at the partition boundaries ride the same sync
  std::vector<int> str_cols;
  if (t) for (int i = 0; i < (int)t->cols.size(); i++) if (t->cols[i]->dtype == B2_STRING) str_cols.push_back(i);
  std::vector<std::vector<int32_t>> str_off(str_cols.size());
  for (size_t k = 0; k < str_cols.size(); k++) {
    const Column* col = t->cols[str_cols[k]];
    str_off[k].resize(W + 1);
    for (int r = 0; r <= W; r++) d2h(&str_off[k][r], col->offsets.as<int32_t>() + offsets[r], 1);
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  std::vector<XHeader> all(W);
  memcpy(all.data(), c->h_all, sizeof(XHeader) * W);
  int anyd = 0, src_schema = -1;
  uint32_t any_null = 0;
  for (int r = 0; r < W; r++) { anyd |= all[r].has_data; any_null |= all[r].nullable_mask; if (src_schema < 0 && all[r].ncols > 0) src_schema = r; }
  c->last_any_more = 0;
  for (int r = 0; r < W; r++) c->last_any_more |= all[r].more;
  *any_data = anyd;
  c->calls++;
  if (!anyd) return B2_OK;
  if (src_schema < 0) throw Error(B2_ERR_INVALID, "exchange: no rank knows the schema");
  if (c->schema_dtype.empty()) {
    c->schema_dtype.assign(all[src_schema].dtype, all[src_schema].dtype + all[src_schema].ncols);
    c->schema_scale.assign(all[src_schema].scale, all[src_schema].scale + all[src_schema].ncols);
  }
  if (!t) { keep.t = empty_table_of(c->schema_dtype, c->schema_scale); t = keep.t; }
  const int ncols = (int)t->cols.size();
  B2_CHECK(offsets[0] == 0 && offsets[W] == t->rows, "offsets must cover the table");
  str_cols.clear();
  for (int i = 0; i < ncols; i++) if (t->cols[i]->dtype == B2_STRING) str_cols.push_back(i);
  if (!mine) { str_off.assign(str_cols.size(), std::vector<int32_t>(W + 1, 0)); }
  const int S = 1 + (int)str_cols.size();
  std::vector<int64_t> send_sz((size_t)W * S, 0);
  for (int r = 0; r < W; r++) {
    send_sz[(size_t)r * S] = offsets[r + 1] - offsets[r];
    for (size_t k = 0; k < str_cols.size(); k++) send_sz[(size_t)r * S + 1 + k] = str_off[k][r + 1] - str_off[k][r];
  }
  // size matrix: all[src][dst][S]
  DevBuf d_send((size_t)W * S * 8), d_sz((size_t)W * W * S * 8);
  h2d(d_send.p, send_sz.data(), send_sz.size());
  NCCL_CHECK(g_nccl.AllGather(d_send.p, d_sz.p, (size_t)W * S * 8, ncclInt8, c->comm, s));
  std::vector<int64_t> szs((size_t)W * W * S);
  d2h(szs.data(), d_sz.p, szs.size());
  sync();
  auto sz = [&](int src, int dst, int k) { return szs[((size_t)src * W + dst) * S + k]; };
  std::vector<int64_t> recv_row_off(W + 1, 0);
  for (int src = 0; src < W; src++) recv_row_off[src + 1] = recv_row_off[src] + sz(src, me, 0);
  const int64_t out_rows = recv_row_off[W];
  if (out_rows > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "exchange result exceeds 2^31-1 rows");

  ColsGuard outs;
  struct Xfer { const char* sbuf; char* rbuf; std::vector<int64_t> soff, roff; int64_t unit; };
  std::vector<Xfer> xfers;
  std::vector<DevBuf> temps;
  std::vector<std::pair<Column*, uint8_t*>> valid_fix;  // (column, received validity bytes)
  std::vector<std::pair<Column*, int32_t*>> str_fix;    // (column, received lengths)
  auto row_xfer = [&](const void* sbuf, void* rbuf, int64_t unit) {
    Xfer x; x.sbuf = (const char*)sbuf; x.rbuf = (char*)rbuf; x.unit = unit;
    for (int r = 0; r <= W; r++) { x.soff.push_back(offsets[r]); x.roff.push_back(recv_row_off[r]); }
    xfers.push_back(std::move(x));
  };
  int sidx = 0;
  int64_t row_bytes = 0;
  for (int i = 0; i < ncols; i++) {
    const Column* ic = t->cols[i];
    std::unique_ptr<Column> oc(new Column());
    oc->dtype = ic->dtype; oc->scale = ic->scale; oc->size = out_rows;
    // validity travels (one byte per row) only for columns that carry NULLs on SOME rank — the grouped send/recv must
    // pair up, so the decision comes from the gathered headers
    if ((any_null >> i) & 1u) {
      oc->valid = DevBuf(validity_bytes(out_rows)); oc->null_count = -1;
      temps.emplace_back((size_t)std::max<int64_t>(t->rows, 1));
      uint8_t* sv = temps.back().as<uint8_t>();
      if (t->rows) launch(bits_to_bytes_kernel, grid_for(t->rows, 256), 256, 0, s, ic->validity(), t->rows, sv);
      temps.emplace_back((size_t)std::max<int64_t>(out_rows, 1));
      uint8_t* rv = temps.back().as<uint8_t>();
      row_xfer(sv, rv, 1);
      valid_fix.push_back({oc.get(), rv});
      row_bytes += 1;
    }
    if (ic->dtype == B2_STRING) {
      temps.emplace_back((size_t)std::max<int64_t>(t->rows, 1) * 4);
      int32_t* slen = temps.back().as<int32_t>();
      if (t->rows) launch(lengths_kernel, grid_for(t->rows, 256), 256, 0, s, ic->offsets.as<int32_t>(), t->rows, slen);
      temps.emplace_back((size_t)(out_rows + 1) * 4);
      int32_t* rlen = temps.back().as<int32_t>();
      row_xfer(slen, rlen, 4);
      int64_t chars = 0;
      Xfer x; x.sbuf = ic->data.as<char>(); x.unit = 1;
      x.soff.resize(W + 1); x.roff.resize(W + 1);
      for (int r = 0; r <= W; r++) x.soff[r] = str_off[sidx][r];
      x.roff[0] = 0;
      for (int src = 0; src < W; src++) { x.roff[src + 1] = x.roff[src] + sz(src, me, 1 + sidx); }
      chars = x.roff[W];
      if (chars > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "exchange result exceeds 2^31-1 chars");
      oc->data = DevBuf((size_t)chars); oc->chars_bytes = chars;
      oc->offsets = DevBuf((size_t)(out_rows + 1) * 4);
      x.rbuf = oc->data.as<char>();
      xfers.push_back(std::move(x));
      str_fix.push_back({oc.get(), rlen});
      sidx++;
      row_bytes += 4;
    } else {
      const int w = dtype_width(ic->dtype);
      oc->data = DevBuf((size_t)out_rows * w);
      row_xfer(ic->data.p, oc->data.p, w);
      row_bytes += w;
    }
    outs.v.push_back(oc.release());
  }
  // one grouped launch: every column slice to every peer (self included: NCCL copies locally)
  {
    KernelTimer kt("nccl_grouped_sendrecv");
    NCCL_CHECK(g_nccl.GroupStart());
    for (auto& x : xfers) {
      for (int r = 0; r < W; r++) {
        const int64_t sb = (x.soff[r + 1] - x.soff[r]) * x.unit, rb = (x.roff[r + 1] - x.roff[r]) * x.unit;
        if (sb) NCCL_CHECK(g_nccl.Send(x.sbuf + x.soff[r] * x.unit, (size_t)sb, ncclInt8, r, c->comm, s));
        if (rb) NCCL_CHECK(g_nccl.Recv(x.rbuf + x.roff[r] * x.unit, (size_t)rb, ncclInt8, r, c->comm, s));
        if (r != me) { c->bytes_sent += sb; c->bytes_received += rb; }
      }
    }
    NCCL_LAUNCH(g_nccl.GroupEnd());
  }
  for (auto& vf : valid_fix) {
    if (out_rows) launch(bytes_to_bits_kernel, grid_for(out_rows, 256), 256, 0, s, vf.second, out_rows, vf.first->valid.as<uint32_t>());
  }
  for (auto& sf : str_fix) exclusive_scan<int32_t, int32_t>(sf.second, sf.first->offsets.as<int32_t>(), out_rows, true);
  sync();  // temps are freed on return
  (void)row_bytes;
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

int b2_exchange(b2_handle comm, b2_handle partitioned_table, const int32_t* offsets, b2_handle* out_table) {
  int32_t any = 0;
  return b2_exchange_ex(comm, partitioned_table, offsets, out_table, &any);
}

// GpuBroadcastExchangeExec (GpuBroadcastExchangeExec.scala: the build side is collected once and every executor gets the
// whole relation): root's table to every rank over ncclBroadcast.  Non-root ranks pass table = 0.
int b2_broadcast_table(b2_handle comm, b2_handle table, int32_t root, b2_handle* out_table) {
  B2_TRY
  Comm* c = comm_from(comm);
  const int W = c->world, me = c->rank;
  B2_CHECK(root >= 0 && root < W, "broadcast root out of range");
  cudaStream_t s = stream();
  Table* t = (me == root) ? table_from(table) : nullptr;
  // header: schema + per-column (rows, chars, nullable)
  struct BHeader { int64_t rows; int32_t ncols; int32_t pad; int32_t dtype[XMAX_COLS], scale[XMAX_COLS]; int64_t chars[XMAX_COLS]; uint32_t nullable_mask; uint32_t pad2; };
  BHeader bh; memset(&bh, 0, sizeof(bh));
  if (t) {
    B2_CHECK((int)t->cols.size() <= XMAX_COLS, "broadcast: more than 32 columns");
    bh.rows = t->rows; bh.ncols = (int)t->cols.size();
    for (int i = 0; i < bh.ncols; i++) {
      const Column* col = t->cols[i];
      bh.dtype[i] = col->dtype; bh.scale[i] = col->scale; bh.chars[i] = col->chars_bytes;
      if (col->nullable()) bh.nullable_mask |= 1u << i;
    }
  }
  DevBuf d_bh(sizeof(BHeader));
  if (t) h2d_bytes(d_bh.p, &bh, sizeof(bh));
  NCCL_LAUNCH(g_nccl.Broadcast(d_bh.p, d_bh.p, sizeof(BHeader), ncclInt8, root, c->comm, s));
  CUDA_CHECK(cudaMemcpyAsync(&bh, d_bh.p, sizeof(bh), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (me == root) { t->refs.fetch_add(1); }
  ColsGuard outs;
  NCCL_CHECK(g_nccl.GroupStart());
  for (int i = 0; i < bh.ncols; i++) {
    Column* oc;
    if (me == root) { oc = t->cols[i]; col_incref(oc); }
    else {
      std::unique_ptr<Column> nc(new Column());
      nc->dtype = bh.dtype[i]; nc->scale = bh.scale[i]; nc->size = bh.rows;
      if (nc->dtype == B2_STRING) { nc->offsets = DevBuf((size_t)(bh.rows + 1) * 4); nc->data = DevBuf((size_t)bh.chars[i]); nc->chars_bytes = bh.chars[i]; }
      else nc->data = DevBuf((size_t)bh.rows * dtype_width(nc->dtype));
      if ((bh.nullable_mask >> i) & 1u) { nc->valid = DevBuf(validity_bytes(bh.rows)); nc->null_count = -1; }
      oc = nc.release();
    }
    outs.v.push_back(oc);
    if (oc->dtype == B2_STRING) {
      NCCL_CHECK(g_nccl.Broadcast(oc->offsets.p, oc->offsets.p, (size_t)(bh.rows + 1) * 4, ncclInt8, root, c->comm, s));
      if (bh.chars[i]) NCCL_CHECK(g_nccl.Broadcast(oc->data.p, oc->data.p, (size_t)bh.chars[i], ncclInt8, root, c->comm, s));
    } else if (bh.rows) {
      NCCL_CHECK(g_nccl.Broadcast(oc->data.p, oc->data.p, (size_t)bh.rows * dtype_width(oc->dtype), ncclInt8, root, c->comm, s));
    }
    if ((bh.nullable_mask >> i) & 1u) NCCL_CHECK(g_nccl.Broadcast(oc->valid.p, oc->valid.p, validity_bytes(bh.rows), ncclInt8, root, c->comm, s));
  }
  NCCL_LAUNCH(g_nccl.GroupEnd());
  if (me == root) table_release(t);
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

}  // extern "C"
