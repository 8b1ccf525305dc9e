// join.cu — a6: hash join build / probe producing gather maps.
// Reference: JoinImpl.innerHashJoin{BuildLeft,BuildRight} -> JoinPrimitives.hashInnerJoin
// (GpuHashJoin.scala:309-409), leftJoin/leftSemi/leftAnti gather maps (:466-600),
// JoinPrimitives.makeLeftOuter/makeSemi/makeAnti (:256-302), null-key rules (:602-640),
// HashJoinIterator (:1374-1553), build-side null filtering (GpuShuffledHashJoinExec.scala:207-212).
//
// The reference API takes both key tables on every call, so the hash table is rebuilt for every
// stream batch.  Here the build side is hashed ONCE into a persistent open-addressing multimap
// (8-byte slots: 32-bit hash tag + 32-bit build row) that any number of probe calls reuse.
// Probe is count -> scan -> write so the gather maps are exactly sized and ordered by stream row.
#include <type_traits>
#include "joinemit.cuh"
#include "prim.cuh"
#include "rowops.cuh"
#include "simplefilter.cuh"

namespace b2 {

Program* program_from(b2_handle h);   // vm.cuh

constexpr uint64_t JSLOT_EMPTY = 0xffffffffffffffffull;

struct JoinTable {
  Table* keys;        // one reference on the build key table
  DevBuf slots;       // uint64 [cap]
  int64_t cap;
  int64_t build_rows;
  bool nulls_equal;
  bool fast = false;      // keys fixed width, <= 8 bytes together, no NULL can match: 16-byte entries {tag|row, packed key}
  bool distinct = false;  // no two build rows share a key (FK -> PK joins): probe is single pass
  // Blocked Bloom filter over the build keys (two bits of one 64-bit word per key, <= 32 MB so that it fits the H100's 50 MB L2
  // while the table itself — 16 B per slot at load <= 0.5 — lives in HBM): a probe row whose key is absent from the build
  // side (most rows of a selective join: TPC-H q3 matches 10-20 %) is rejected by ONE L2 hit instead of a random HBM
  // access into the table.  Same idea as the runtime Bloom filter Spark injects in front of such joins
  // (GpuBloomFilterMightContain in the reference), applied inside the probe.
  DevBuf bloom;
  uint32_t bloom_mask = 0;  // 64-bit words - 1; 0 = no filter
  std::vector<int> key_idx;
  ~JoinTable() { if (keys) table_release(keys); }
};

__device__ __forceinline__ bool any_null_key(const KeyCols& k, int64_t r) {
  for (int i = 0; i < k.n; i++) if (!row_valid(k.c[i].valid, r)) return true;
  return false;
}

__device__ __forceinline__ uint64_t pack_join_key(const KeyCols& ks, int64_t r) {
  uint64_t bits = 0; int shift = 0;
  for (int i = 0; i < ks.n; i++) { bits |= key_bits(ks.c[i], r) << shift; shift += 8 * ks.c[i].width; }
  return bits;
}
__device__ __forceinline__ uint32_t hash_packed(uint64_t kb) { const uint64_t h = mix64(kb ^ 0x9e3779b97f4a7c15ull); return (uint32_t)(h ^ (h >> 32)); }

// bloom_mask: bits 0..27 = words - 1, bits 28..29 = extra bits set per key beyond the first two (k = 2..4)
__device__ __forceinline__ void bloom_of(uint32_t h, uint32_t bloom_mask, uint32_t& word, unsigned long long& bits) {
  const uint64_t p = (uint64_t)h * 0x9E3779B97F4A7C15ull;
  word = (uint32_t)(p >> 40) & (bloom_mask & 0x0fffffffu);
  bits = (1ull << ((p >> 8) & 63)) | (1ull << ((p >> 14) & 63));
  const uint32_t extra = bloom_mask >> 28;
  if (extra >= 1) bits |= 1ull << ((p >> 20) & 63);
  if (extra >= 2) bits |= 1ull << ((p >> 26) & 63);
}
__device__ __forceinline__ bool bloom_may_contain(const unsigned long long* __restrict__ bloom, uint32_t bloom_mask, uint32_t h) {
  if (!bloom) return true;
  uint32_t w; unsigned long long bits;
  bloom_of(h, bloom_mask, w, bits);
  return (__ldg(&bloom[w]) & bits) == bits;
}

__global__ void join_build_kernel(const __grid_constant__ KeyCols keys, int64_t n, uint64_t* __restrict__ slots,
                                  uint32_t mask, bool nulls_equal, bool fast, int32_t* __restrict__ has_dups,
                                  unsigned long long* __restrict__ bloom, uint32_t bloom_mask) {
  const int sh = fast ? 1 : 0;  // entry stride: 2 words when the packed key rides along
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    if (!nulls_equal && any_null_key(keys, r)) continue;  // a NULL key can never match: keep it out of the table
    uint64_t kb = 0;
    uint32_t h;
    if (fast) { kb = pack_join_key(keys, r); h = hash_packed(kb); } else h = row_hash(keys, r);
    const uint64_t entry = ((uint64_t)h << 32) | (uint32_t)r;
    if (bloom) { uint32_t w; unsigned long long bits; bloom_of(h, bloom_mask, w, bits); atomicOr(&bloom[w], bits); }
    uint32_t idx = h & mask;
    while (true) {
      unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&slots[(size_t)idx << sh]), (unsigned long long)JSLOT_EMPTY, (unsigned long long)entry);
      if (old == JSLOT_EMPTY) { if (fast) slots[((size_t)idx << 1) + 1] = kb; break; }
      // occupied: a slot with my tag may hold my key -> the build side is not distinct
      if ((uint32_t)(old >> 32) == h && *has_dups == 0 && rows_equal(keys, r, keys, (int32_t)(uint32_t)old, nulls_equal)) atomicExch(has_dups, 1);
      idx = (idx + 1) & mask;
    }
  }
}

// one probe step: entry word (and, for packed keys, the key from the same 16-byte line)
__device__ __forceinline__ uint64_t join_entry(const uint64_t* __restrict__ slots, uint32_t idx, bool fast, uint64_t& key) {
  if (fast) { const ulonglong2 e = *reinterpret_cast<const ulonglong2*>(&slots[(size_t)idx << 1]); key = e.y; return e.x; }
  key = 0;
  return slots[idx];
}

// Matched build rows across stream batches (RIGHT OUTER, and FULL OUTER with a condition): a JoinTracker holds one bit per build
// row of one hash table, and the tracking (TRACK) probe variants set bit br where they find build row br — inside the probe,
// where the reference filters the gather map, copies it, scatters it into a BOOL8 tracker and rebuilds the tracker per batch
// (HashJoinStreamSideIterator.updateTrackingMask, GpuHashJoin.scala:2164-2204).  The word is read first and the atomic issued
// only when the bit is clear: in FK -> PK joins many stream rows hit the same build row, and neighbouring build rows share a word.
__device__ __forceinline__ void track_hit(uint32_t* __restrict__ bits, int32_t br) {
  uint32_t* w = bits + ((uint32_t)br >> 5);
  const uint32_t b = 1u << (br & 31);
  if (!(*w & b)) atomicOr(w, b);
}

// single pass for a distinct build side: at most one match per stream row.
//   INNER: pairs appended with ONE atomic per warp and PI x 32 rows (join output order is unspecified: docs/compatibility.md:18-25)
//   LEFT OUTER: row r -> (r, match or INT32_MIN), no compaction at all
// Each warp owns chunks of PI x 32 consecutive rows and works on them in phases, so that every lane has PI independent
// loads in flight at each step (selection vector -> keys -> Bloom words -> table slots) instead of one dependent chain, and
// the output range of a whole chunk is reserved with a single atomic (the per-32-rows atomic on one address was the
// serialisation point of the kernel: ~10 M same-address atomics per TPC-H q3 step).
constexpr int PI = 8;
template <bool TRACK>
__global__ void __launch_bounds__(256) join_probe_distinct_kernel(const __grid_constant__ KeyCols probe, const __grid_constant__ KeyCols build, int64_t n,
                                           const uint64_t* __restrict__ slots, uint32_t mask, bool nulls_equal,
                                           bool fast, int kind, unsigned long long* __restrict__ total, int32_t* __restrict__ left_map,
                                           int32_t* __restrict__ right_map, const unsigned long long* __restrict__ bloom, uint32_t bloom_mask,
                                           const int32_t* __restrict__ sel, uint32_t* __restrict__ track) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * (32 * PI); base < n; base += nwarps * (32 * PI)) {
    int64_t src[PI];
    uint64_t kb[PI];
    uint32_t h[PI];
    bool live[PI];
    int32_t br[PI];
    // selection vector: probe row rr of the (virtual) filtered batch is row sel[rr] of the batch itself; the left map then
    // carries ORIGINAL row ids, so the payload gather reads the unfiltered batch and no filtered copy ever exists
#pragma unroll
    for (int j = 0; j < PI; j++) {
      const int64_t rr = base + j * 32 + lane;
      src[j] = rr < n ? (sel ? (int64_t)sel[rr] : rr) : -1;
    }
#pragma unroll
    for (int j = 0; j < PI; j++) {
      br[j] = INT32_MIN; kb[j] = 0; h[j] = 0;
      live[j] = src[j] >= 0 && ((nulls_equal && !fast) || !any_null_key(probe, src[j]));  // fast: the build side holds no NULL keys, so a NULL probe key matches nothing
      if (live[j]) { if (fast) { kb[j] = pack_join_key(probe, src[j]); h[j] = hash_packed(kb[j]); } else h[j] = row_hash(probe, src[j]); }
    }
    if (bloom) {
      unsigned long long w[PI];
#pragma unroll
      for (int j = 0; j < PI; j++) {
        uint32_t wi = 0; unsigned long long bits = 0;
        bloom_of(h[j], bloom_mask, wi, bits);
        w[j] = live[j] ? __ldg(&bloom[wi]) : 0ull;
        kb[j] = fast ? kb[j] : 0;
        live[j] = live[j] && (w[j] & bits) == bits;
      }
    }
#pragma unroll
    for (int j = 0; j < PI; j++) {
      if (!live[j]) continue;
      uint32_t idx = h[j] & mask;
      while (true) {
        uint64_t ek;
        const uint64_t e = join_entry(slots, idx, fast, ek);
        if (e == JSLOT_EMPTY) break;
        if ((uint32_t)(e >> 32) == h[j]) {
          const bool eq = fast ? (ek == kb[j]) : rows_equal(probe, src[j], build, (int32_t)(uint32_t)e, nulls_equal);
          if (eq) { br[j] = (int32_t)(uint32_t)e; break; }
        }
        idx = (idx + 1) & mask;
      }
    }
    if constexpr (TRACK) {
#pragma unroll
      for (int j = 0; j < PI; j++) if (br[j] != INT32_MIN) track_hit(track, br[j]);
    }
    if (kind == B2_JOIN_LEFT_OUTER) {
#pragma unroll
      for (int j = 0; j < PI; j++) {
        const int64_t rr = base + j * 32 + lane;
        if (rr < n) { left_map[rr] = (int32_t)src[j]; right_map[rr] = br[j]; }
      }
    } else {
      uint32_t ball[PI];
      uint32_t hits = 0;
#pragma unroll
      for (int j = 0; j < PI; j++) { ball[j] = __ballot_sync(0xffffffffu, br[j] != INT32_MIN); hits += __popc(ball[j]); }
      unsigned long long o = 0;
      if (lane == 0 && hits) o = atomicAdd(total, (unsigned long long)hits);
      o = __shfl_sync(0xffffffffu, o, 0);
#pragma unroll
      for (int j = 0; j < PI; j++) {
        if (br[j] != INT32_MIN) { const unsigned long long at = o + __popc(ball[j] & ((1u << lane) - 1u)); left_map[at] = (int32_t)src[j]; right_map[at] = br[j]; }
        o += __popc(ball[j]);
      }
    }
  }
}

// Keeps a region (the Bloom filter) in the persisting part of L2 while probe kernels stream the probe columns past it
// (cudaStreamAttributeAccessPolicyWindow); off unless B2_JOIN_BLOOM_PERSIST is set.
struct L2Persist {
  bool on = false;
  L2Persist(void* p, size_t bytes) {
    static const bool enabled = getenv("B2_JOIN_BLOOM_PERSIST") != nullptr;
    if (!enabled || !p || !bytes) return;
    static size_t max_window = 0, carve = 0;
    static bool init = false;
    if (!init) {
      init = true;
      int dev = 0; cudaGetDevice(&dev);
      cudaDeviceProp prop; cudaGetDeviceProperties(&prop, dev);
      carve = std::min<size_t>((size_t)prop.persistingL2CacheMaxSize, (size_t)48 << 20);
      max_window = (size_t)prop.accessPolicyMaxWindowSize;
      if (carve) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve);
    }
    if (!carve || !max_window) return;
    cudaStreamAttrValue a; memset(&a, 0, sizeof(a));
    a.accessPolicyWindow.base_ptr = p;
    a.accessPolicyWindow.num_bytes = std::min(bytes, max_window);
    a.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)carve / (double)a.accessPolicyWindow.num_bytes);
    a.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    a.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    on = cudaStreamSetAttribute(stream(), cudaStreamAttributeAccessPolicyWindow, &a) == cudaSuccess;
    if (!on) cudaGetLastError();
  }
  ~L2Persist() {
    if (!on) return;
    cudaStreamAttrValue a; memset(&a, 0, sizeof(a));
    a.accessPolicyWindow.num_bytes = 0;
    cudaStreamSetAttribute(stream(), cudaStreamAttributeAccessPolicyWindow, &a);
  }
};

// The commonest probe of all — INNER join against a distinct build side on ONE integer key column without NULLs (every
// FK -> PK join of TPC-H) — without the generic row machinery (KeyCols loops, validity, runtime join kind): ~6x fewer
// instructions per row than join_probe_distinct_kernel.  A warp takes PQ x 32 rows at a time (probe_distinct1_rows):
//   1. keys, then Bloom words: PQ independent loads per lane at each step;
//   2. the rows that pass the Bloom filter (10-20 % in q3) are compacted into a per-warp queue in shared memory, so the
//      random HBM accesses into the table are issued by FULL warps in one or two rounds (the generic kernel walked its 8 row
//      slots one after the other, each round with 2-3 live lanes paying a full memory latency);
//   3. one output reservation (atomic) per round; each round's hits are written in ascending row order when r[] ascends
//      (j-major, then lane), so the payload gathers read the batch in order.
// (Tried and measured slower on the q3 step: evict-first loads of the selection vector and the key column plus
// evict-last Bloom words.  Unlike part_scatter2 — hash.cu — nothing here is half-written and waiting in L2.)
constexpr int PQ = 8;

// The output row descriptors of the emitting probe (EMIT): instead of the gather maps, a lane that finds build row br for
// stream row src writes the joined row itself at the offset it reserved — the stream columns loaded at src (the key column
// from the probed key, no load), the build columns unpacked from one aligned 8- or 16-byte load of the packed payload at br
// (JoinPayload).  Offsets at or past `cap` are counted and not written: the caller sizes the output from an estimate and
// redoes the batch through the maps when the total passes it.
constexpr int EM_STREAM = 3, EM_BUILD = 4;   // columns per side (a fourth stream column spills)
struct EmitCols {
  int32_t ns, nb, pw;                  // stream columns, build columns, payload bytes per build row (0, 8 or 16)
  int8_t s_w[EM_STREAM];
  int8_t b_w[EM_BUILD], b_off[EM_BUILD];   // width and byte offset in the payload row
  const void* s_in[EM_STREAM];         // nullptr: the join key
  void* s_out[EM_STREAM];
  void* b_out[EM_BUILD];
  const void* packed;
  unsigned long long cap;              // rows allocated in every output column
};
struct NoEmit {};

// Columns of 4, 8 (and, on the build side, 16) bytes only: every further width is one more branch per column, and those
// branches cost the emitting kernel registers it does not have under __launch_bounds__(SF_NT, FP_CTAS) (it spilled)
__host__ __device__ __forceinline__ bool emit_width_ok(int w, bool build) { return w == 4 || w == 8 || (build && w == 16); }
// every load first, then the stores: the loads are independent random accesses, and the stores could alias them
__device__ __forceinline__ void emit_row(const EmitCols& em, uint32_t o, int32_t src, uint64_t kb, int32_t br) {   // o < cap < 2^31
  uint64_t v[EM_STREAM];
#pragma unroll
  for (int c = 0; c < EM_STREAM; c++) {
    v[c] = kb;
    if (c < em.ns && em.s_in[c])
      v[c] = em.s_w[c] == 8 ? __ldg(reinterpret_cast<const unsigned long long*>(em.s_in[c]) + src) : __ldg(reinterpret_cast<const uint32_t*>(em.s_in[c]) + src);
  }
  uint64_t lo = 0, hi = 0;
  if (em.pw == 16) { const ulonglong2 b = __ldg(reinterpret_cast<const ulonglong2*>(em.packed) + br); lo = b.x; hi = b.y; }
  else if (em.pw == 8) lo = __ldg(reinterpret_cast<const unsigned long long*>(em.packed) + br);
#pragma unroll
  for (int c = 0; c < EM_STREAM; c++) {
    if (c >= em.ns) break;
    if (em.s_w[c] == 8) reinterpret_cast<unsigned long long*>(em.s_out[c])[o] = v[c];
    else reinterpret_cast<uint32_t*>(em.s_out[c])[o] = (uint32_t)v[c];
  }
#pragma unroll
  for (int c = 0; c < EM_BUILD; c++) {
    if (c >= em.nb) break;
    const int off = em.b_off[c];
    const uint64_t x = off & 8 ? hi : lo;
    if (em.b_w[c] == 16) reinterpret_cast<ulonglong2*>(em.b_out[c])[o] = make_ulonglong2(lo, hi);
    else if (em.b_w[c] == 8) reinterpret_cast<unsigned long long*>(em.b_out[c])[o] = x;
    else reinterpret_cast<uint32_t*>(em.b_out[c])[o] = off & 4 ? (uint32_t)(x >> 32) : (uint32_t)x;
  }
}

template <typename K, bool TRACK, bool EMIT = false>
__device__ __forceinline__ void probe_distinct1_rows(const K* __restrict__ keys, const int32_t (&r)[PQ], const uint64_t* __restrict__ slots,
                                                     uint32_t mask, const unsigned long long* __restrict__ bloom, uint32_t bloom_mask,
                                                     unsigned long long* __restrict__ total, int32_t* __restrict__ left_map,
                                                     int32_t* __restrict__ right_map, int32_t* s_q, uint32_t* __restrict__ track,
                                                     const EmitCols* em = nullptr) {
  typedef typename std::make_unsigned<K>::type UK;
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t pass = 0;
  if (bloom) {
    uint32_t h[PQ];
    unsigned long long wv[PQ];
#pragma unroll
    for (int j = 0; j < PQ; j++) h[j] = r[j] >= 0 ? hash_packed((uint64_t)(UK)keys[r[j]]) : 0u;
#pragma unroll
    for (int j = 0; j < PQ; j++) {
      uint32_t wi; unsigned long long bits;
      bloom_of(h[j], bloom_mask, wi, bits);
      wv[j] = r[j] >= 0 ? __ldg(&bloom[wi]) : 0ull;
    }
#pragma unroll
    for (int j = 0; j < PQ; j++) {
      uint32_t wi; unsigned long long bits;
      bloom_of(h[j], bloom_mask, wi, bits);
      pass |= (uint32_t)(r[j] >= 0 && (wv[j] & bits) == bits) << j;
    }
  } else {
#pragma unroll
    for (int j = 0; j < PQ; j++) pass |= (uint32_t)(r[j] >= 0) << j;
  }
  int qn = 0;
#pragma unroll
  for (int j = 0; j < PQ; j++) {
    const bool p = (pass >> j) & 1u;
    const uint32_t b = __ballot_sync(0xffffffffu, p);
    if (p) s_q[qn + __popc(b & lt)] = r[j];
    qn += __popc(b);
  }
  __syncwarp();
  for (int q0 = 0; q0 < qn; q0 += 32) {
    const int q = q0 + lane;
    int32_t br = INT32_MIN, src = 0;
    uint64_t key = 0;   // EMIT: the key column's value
    if (q < qn) {
      src = s_q[q];
      const uint64_t kb = (uint64_t)(UK)keys[src];
      const uint32_t hh = hash_packed(kb);
      uint32_t idx = hh & mask;
      key = kb;
      while (true) {
        const ulonglong2 e = *reinterpret_cast<const ulonglong2*>(&slots[(size_t)idx << 1]);
        if (e.x == JSLOT_EMPTY) break;
        if ((uint32_t)(e.x >> 32) == hh && e.y == kb) { br = (int32_t)(uint32_t)e.x; break; }
        idx = (idx + 1) & mask;
      }
    }
    const bool hit = br != INT32_MIN;
    const uint32_t b = __ballot_sync(0xffffffffu, hit);
    if (b) {
      unsigned long long o = 0;
      if (lane == 0) o = atomicAdd(total, (unsigned long long)__popc(b));
      o = __shfl_sync(0xffffffffu, o, 0) + __popc(b & lt);
      if constexpr (EMIT) {
        if (hit && o < em->cap) emit_row(*em, (uint32_t)o, src, key, br);
      } else if (hit) {
        left_map[o] = src; right_map[o] = br;
        if constexpr (TRACK) track_hit(track, br);
      }
    }
  }
  __syncwarp();   // the queue is rewritten by the next call
}

// every row of the batch (SEL = false) or the rows of a selection vector (a filter below the join emitted row ids)
template <typename K, bool SEL, bool TRACK>
__global__ void __launch_bounds__(256) join_probe_distinct1_kernel(const K* __restrict__ keys, const int32_t* __restrict__ sel, int64_t n,
                                                                   const uint64_t* __restrict__ slots, uint32_t mask,
                                                                   const unsigned long long* __restrict__ bloom, uint32_t bloom_mask,
                                                                   unsigned long long* __restrict__ total, int32_t* __restrict__ left_map,
                                                                   int32_t* __restrict__ right_map, uint32_t* __restrict__ track) {
  __shared__ int32_t s_q[8][32 * PQ];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * (32 * PQ); base < n; base += nwarps * (32 * PQ)) {
    int32_t r[PQ];
#pragma unroll
    for (int j = 0; j < PQ; j++) {
      const int64_t rr = base + j * 32 + lane;
      r[j] = rr < n ? (SEL ? sel[rr] : (int32_t)rr) : -1;
    }
    probe_distinct1_rows<K, TRACK>(keys, r, slots, mask, bloom, bloom_mask, total, left_map, right_map, s_q[w], track);
  }
}

// A simple filter (simplefilter.cuh) directly below the stream side, evaluated inside the probe: no selection vector is
// written, copied back or re-read.  Per tile of FP_TILE consecutive rows:
//   1. sf_tile streams the predicate columns (16-byte loads, the selection-vector kernel's code) into a bit mask in shared
//      memory;
//   2. the passing rows become a dense, ascending queue of tile offsets in shared memory (one mask word per thread, block
//      scan of the popcounts; the join output is unordered, so no look-back across tiles);
//   3. full warps take the queue PQ x 32 ids at a time through probe_distinct1_rows.  Lanes only load keys of passing rows:
//      the same sectors the selection-vector path reads.
// The probe is bound by latency per row slot, not by bytes, so the queue is what makes the fusion pay: walking every row
// through the dependent chain (predicate -> key -> Bloom word) would leave the lanes of failing rows idle at every step
// (about half of them on q3's date filters).  The streaming of one CTA overlaps the lookups of the others (FP_CTAS per SM;
// 3 measured slower, 5 spills).
constexpr int FP_TILE = 8 * 1024, FP_WORDS = FP_TILE / 32, FP_CTAS = 4;
static_assert(FP_WORDS == SF_NT, "one mask word per thread");
// EMIT: the output rows are written (EmitCols `em`) instead of the maps, which are then null
template <typename K, bool TRACK, bool EMIT = false>
__global__ void __launch_bounds__(SF_NT, FP_CTAS) join_filter_probe_kernel(const __grid_constant__ SimplePred sp, const K* __restrict__ keys, int64_t n,
                                                                          const uint64_t* __restrict__ slots, uint32_t mask,
                                                                          const unsigned long long* __restrict__ bloom, uint32_t bloom_mask,
                                                                          unsigned long long* __restrict__ total, int32_t* __restrict__ left_map,
                                                                          int32_t* __restrict__ right_map, unsigned long long* __restrict__ npass,
                                                                          uint32_t* __restrict__ track,
                                                                          const __grid_constant__ typename std::conditional<EMIT, EmitCols, NoEmit>::type em) {
  __shared__ uint32_t s_mask[FP_WORDS];
  __shared__ uint16_t s_rows[FP_TILE];               // offsets in the tile of the passing rows, ascending
  __shared__ int32_t s_q[SF_NT / 32][32 * PQ];
  __shared__ uint32_t s_wtot[SF_NT / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ntiles = (n + FP_TILE - 1) / FP_TILE;
  // a 32-bit tile index in the emitting variant (n < 2^31): the 64-bit one is the register it would otherwise spill; the maps
  // variants keep theirs, and with it their code
  typedef typename std::conditional<EMIT, int32_t, int64_t>::type TileIdx;
  for (TileIdx tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = (int64_t)tile * FP_TILE;
    sf_tile(sp, row0, (int)min((int64_t)FP_TILE, n - row0), s_mask, FP_WORDS);
    const uint32_t m = s_mask[threadIdx.x], c = __popc(m);
    uint32_t inc = c;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
    if (lane == 31) s_wtot[w] = inc;
    __syncthreads();
    uint32_t pos = inc - c;
    int qn = 0;
#pragma unroll
    for (int i = 0; i < SF_NT / 32; i++) { const uint32_t x = s_wtot[i]; pos += i < w ? x : 0u; qn += (int)x; }
    for (uint32_t mm = m; mm; mm &= mm - 1) s_rows[pos++] = (uint16_t)(threadIdx.x * 32 + __ffs(mm) - 1);
    if (threadIdx.x == 0 && qn) atomicAdd(npass, (unsigned long long)qn);
    __syncthreads();
    for (int q0 = w * 32 * PQ; q0 < qn; q0 += SF_NT * PQ) {
      int32_t r[PQ];
#pragma unroll
      for (int j = 0; j < PQ; j++) {
        const int q = q0 + j * 32 + lane;
        r[j] = q < qn ? (int32_t)(row0 + s_rows[q]) : -1;
      }
      if constexpr (EMIT) probe_distinct1_rows<K, TRACK, true>(keys, r, slots, mask, bloom, bloom_mask, total, left_map, right_map, s_q[w], track, &em);
      else probe_distinct1_rows<K, TRACK>(keys, r, slots, mask, bloom, bloom_mask, total, left_map, right_map, s_q[w], track);
    }
    __syncthreads();   // s_mask, s_rows and s_wtot are rewritten by the next tile
  }
}

// MODE 0: count matches per probe row; MODE 1: write pairs at offsets (TRACK: and mark the build rows)
template <int MODE, bool TRACK = false>
__global__ void join_probe_kernel(const __grid_constant__ KeyCols probe, const __grid_constant__ KeyCols build, int64_t n,
                                  const uint64_t* __restrict__ slots, uint32_t mask, bool nulls_equal,
                                  bool fast, int kind, int32_t* __restrict__ counts, const int64_t* __restrict__ offsets,
                                  int32_t* __restrict__ left_map, int32_t* __restrict__ right_map,
                                  const unsigned long long* __restrict__ bloom, uint32_t bloom_mask, const int32_t* __restrict__ sel,
                                  uint32_t* __restrict__ track) {
  for (int64_t rr = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; rr < n; rr += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = sel ? (int64_t)sel[rr] : rr;   // see join_probe_distinct_kernel
    int32_t matches = 0;
    int64_t o = MODE == 1 ? offsets[rr] : 0;
    const bool semi_like = kind == B2_JOIN_LEFT_SEMI || kind == B2_JOIN_LEFT_ANTI;
    if ((nulls_equal && !fast) || !any_null_key(probe, r)) {  // fast: see join_probe_distinct_kernel
      uint64_t kb = 0;
      uint32_t h;
      if (fast) { kb = pack_join_key(probe, r); h = hash_packed(kb); } else h = row_hash(probe, r);
      uint32_t idx = h & mask;
      const bool maybe = bloom_may_contain(bloom, bloom_mask, h);
      while (maybe) {
        uint64_t ek;
        const uint64_t e = join_entry(slots, idx, fast, ek);
        if (e == JSLOT_EMPTY) break;
        if ((uint32_t)(e >> 32) == h) {
          const int32_t br = (int32_t)(uint32_t)e;
          if (fast ? (ek == kb) : rows_equal(probe, r, build, br, nulls_equal)) {
            if (MODE == 1 && !semi_like) {
              left_map[o + matches] = (int32_t)r; right_map[o + matches] = br;
              if constexpr (TRACK) track_hit(track, br);
            }
            matches++;
            if (semi_like) break;
          }
        }
        idx = (idx + 1) & mask;
      }
    }
    int32_t emit;
    switch (kind) {
      case B2_JOIN_INNER: emit = matches; break;
      case B2_JOIN_LEFT_OUTER: emit = matches > 0 ? matches : 1; break;
      case B2_JOIN_LEFT_SEMI: emit = matches > 0 ? 1 : 0; break;
      default: emit = matches > 0 ? 0 : 1; break;  // LEFT_ANTI
    }
    if (MODE == 0) counts[rr] = emit;
    else {
      if (semi_like) { if (emit) left_map[o] = (int32_t)r; }
      else if (kind == B2_JOIN_LEFT_OUTER && matches == 0) { left_map[o] = (int32_t)r; right_map[o] = INT32_MIN; }
    }
  }
}

// ---- the tracker's other two kernels: marking through a gather map, and the ids of the clear bits -------------------
// tracker_mark_kernel: bit right_map[i] for every i whose pass[i] is true (BOOL8, NULL = false; no pass = every i).  Negative
// entries (INT32_MIN, OutOfBoundsPolicy.NULLIFY) are skipped; an entry >= nb sets *bad.  Serves conditional joins, where only
// the pairs that pass the condition count.
__global__ void tracker_mark_kernel(const int32_t* __restrict__ right_map, const int8_t* __restrict__ pass, const uint32_t* __restrict__ pass_valid,
                                    int64_t n, int64_t nb, uint32_t* __restrict__ bits, int32_t* __restrict__ bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t r = right_map[i];
    if (r < 0 || (pass && !(pass[i] && row_valid(pass_valid, i)))) continue;
    if (r >= nb) { *bad = 1; continue; }
    track_hit(bits, r);
  }
}

// tracker_unmatched (HashOuterJoinIterator.getFinalBatch, GpuHashJoin.scala:2288-2326): the bitmap -> ascending INT32 ids of
// its clear bits.  A tile is TU_NT x TU_WPT words (65536 build rows); count pass (popcount of the complemented words, tail word
// masked) -> exclusive_scan of the tile counts -> write pass.  In the write pass warp w of a tile owns 32 x TU_WPT consecutive
// words and takes them 32 at a time (lane = word, so the ids come out ascending); a round's ids (<= 1024) are staged in shared
// memory and leave as aligned 16-byte vectors.  Bytes: nb / 8 read twice, 4 per unmatched row written (8 with `left_fill`).
constexpr int TU_NT = 256, TU_WPT = 8, TU_TILE = TU_NT * TU_WPT;
__device__ __forceinline__ uint32_t clear_bits(const uint32_t* __restrict__ bits, int64_t i, int64_t nwords, uint32_t tail) {
  if (i >= nwords) return 0u;
  const uint32_t m = ~bits[i];
  return i == nwords - 1 ? m & tail : m;
}
__global__ void __launch_bounds__(TU_NT) tracker_count_kernel(const uint32_t* __restrict__ bits, int64_t nwords, uint32_t tail,
                                                              int32_t* __restrict__ counts) {
  __shared__ int32_t s_w[TU_NT / 32];
  const int64_t w0 = (int64_t)blockIdx.x * TU_TILE;
  int c = 0;
#pragma unroll
  for (int j = 0; j < TU_WPT; j++) c += __popc(clear_bits(bits, w0 + j * TU_NT + threadIdx.x, nwords, tail));
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
#pragma unroll
    for (int k = 0; k < TU_NT / 32; k++) t += s_w[k];
    counts[blockIdx.x] = t;
  }
}
// the warp's `cnt` staged values to dst[0..cnt): single elements up to the first 16-byte boundary of dst, then aligned
// vectors, then the tail (dst 4-byte aligned)
template <typename V>
__device__ __forceinline__ void warp_store_aligned(int32_t* __restrict__ dst, int cnt, int lane, V&& value) {
  const int head = min(cnt, (int)(((16 - ((uintptr_t)dst & 15)) & 15) >> 2));
  for (int k = lane; k < head; k += 32) dst[k] = value(k);
  const int nv = (cnt - head) >> 2;
  for (int v = lane; v < nv; v += 32) {
    const int k = head + 4 * v;
    *reinterpret_cast<int4*>(dst + k) = make_int4(value(k), value(k + 1), value(k + 2), value(k + 3));
  }
  for (int k = head + 4 * nv + lane; k < cnt; k += 32) dst[k] = value(k);
}
__global__ void __launch_bounds__(TU_NT) tracker_write_kernel(const uint32_t* __restrict__ bits, int64_t nwords, uint32_t tail,
                                                              const int32_t* __restrict__ offs, int32_t* __restrict__ ids,
                                                              int32_t* __restrict__ left_fill) {
  __shared__ int32_t s_stage[TU_NT / 32][32 * 32];
  __shared__ int32_t s_wt[TU_NT / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t w0 = (int64_t)blockIdx.x * TU_TILE + w * (32 * TU_WPT);   // this warp's first word
  uint32_t m[TU_WPT];
  int tot = 0;
#pragma unroll
  for (int j = 0; j < TU_WPT; j++) { m[j] = clear_bits(bits, w0 + j * 32 + lane, nwords, tail); tot += __popc(m[j]); }
  tot = __reduce_add_sync(0xffffffffu, tot);
  if (lane == 0) s_wt[w] = tot;
  __syncthreads();
  int64_t g = offs[blockIdx.x];
  for (int k = 0; k < w; k++) g += s_wt[k];
  int32_t* st = s_stage[w];
#pragma unroll
  for (int j = 0; j < TU_WPT; j++) {
    const int c = __popc(m[j]);
    int inc = c;
    for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
    const int cnt = __shfl_sync(0xffffffffu, inc, 31);
    if (cnt == 0) continue;
    int pos = inc - c;
    const int32_t row0 = (int32_t)((w0 + j * 32 + lane) * 32);
    for (uint32_t mm = m[j]; mm; mm &= mm - 1) st[pos++] = row0 + __ffs(mm) - 1;
    __syncwarp();
    warp_store_aligned(ids + g, cnt, lane, [&](int k) { return st[k]; });
    if (left_fill) warp_store_aligned(left_fill + g, cnt, lane, [](int) { return INT32_MIN; });
    __syncwarp();   // the stage is rewritten by the next round
    g += cnt;
  }
}

struct JoinTracker {
  const void* table;   // the JoinTable whose build rows the bits stand for
  int64_t nb;
  DevBuf bits;         // uint32 [ceil(nb / 32)], zeroed at creation
  DevBuf bad;          // int32: tracker_mark_kernel saw an entry >= nb
};
static JoinTracker* tracker_new(const void* table, int64_t nb) {
  std::unique_ptr<JoinTracker> tr(new JoinTracker());
  tr->table = table; tr->nb = nb;
  tr->bits = DevBuf((size_t)std::max<int64_t>((nb + 31) / 32, 1) * 4);
  tr->bad = DevBuf(4);
  CUDA_CHECK(cudaMemsetAsync(tr->bits.p, 0, tr->bits.bytes, stream()));
  CUDA_CHECK(cudaMemsetAsync(tr->bad.p, 0, 4, stream()));
  return tr.release();
}
static void tracker_mark(JoinTracker* tr, const int32_t* right_map, int64_t n, const Column* pass) {
  if (n)
    launch("tracker_mark_kernel", tracker_mark_kernel, grid_for(n, 256), 256, 0, stream(), right_map, pass ? pass->data.as<int8_t>() : nullptr,
           pass ? pass->validity() : nullptr, n, tr->nb, tr->bits.as<uint32_t>(), tr->bad.as<int32_t>());
}
// count pass + scan: the number of clear bits; `offs` keeps the tile offsets for tracker_unmatched_write
static int64_t tracker_unmatched_count(const JoinTracker* tr, DevBuf& offs) {
  const int64_t nwords = (tr->nb + 31) / 32, ntiles = (nwords + TU_TILE - 1) / TU_TILE;
  offs = DevBuf((size_t)(ntiles + 1) * 4);
  if (!ntiles) return 0;
  const uint32_t tail = (tr->nb & 31) ? (1u << (tr->nb & 31)) - 1u : 0xffffffffu;
  launch("tracker_count_kernel", tracker_count_kernel, (int)ntiles, TU_NT, 0, stream(), tr->bits.as<uint32_t>(), nwords, tail, offs.as<int32_t>());
  exclusive_scan<int32_t, int32_t>(offs.as<int32_t>(), offs.as<int32_t>(), ntiles, true);
  int32_t u = 0;
  d2h(&u, offs.as<int32_t>() + ntiles, 1);
  sync();
  return u;
}
// write pass: the ascending ids to ids[0..u), and INT32_MIN to left_fill[0..u) when given
static void tracker_unmatched_write(const JoinTracker* tr, const DevBuf& offs, int64_t u, int32_t* ids, int32_t* left_fill) {
  if (!u) return;
  const int64_t nwords = (tr->nb + 31) / 32, ntiles = (nwords + TU_TILE - 1) / TU_TILE;
  const uint32_t tail = (tr->nb & 31) ? (1u << (tr->nb & 31)) - 1u : 0xffffffffu;
  launch("tracker_write_kernel", tracker_write_kernel, (int)ntiles, TU_NT, 0, stream(), tr->bits.as<uint32_t>(), nwords, tail, offs.as<int32_t>(), ids,
         left_fill);
}

// ---- mixed (conditional) joins: which stream rows own at least one pair that passes the join condition ------------------------
__global__ void mark_passing_kernel(const int32_t* __restrict__ left_map, const int8_t* __restrict__ pass, const uint32_t* __restrict__ pass_valid, int64_t n,
                                    int8_t* __restrict__ flags) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (pass[i] && row_valid(pass_valid, i)) flags[left_map[i]] = 1;
}
__global__ void invert_flags_kernel(int8_t* __restrict__ flags, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) flags[i] = flags[i] ? 0 : 1;
}
// BOOL8 column over the stream rows: 1 where some (stream row, build row) pair of the equi-join passed the condition
// (invert: 1 where none did)
Column* rows_with_passing_pair(const Column* left_map, const Column* pass, int64_t stream_rows, bool invert) {
  ColGuard flags(new_column(B2_BOOL8, 0, stream_rows, false));
  if (stream_rows) CUDA_CHECK(cudaMemsetAsync(flags.c->data.p, 0, (size_t)stream_rows, stream()));
  if (left_map->size)
    launch(mark_passing_kernel, grid_for(left_map->size, 256), 256, 0, stream(), left_map->data.as<int32_t>(), pass->data.as<int8_t>(), pass->validity(),
           left_map->size, flags.c->data.as<int8_t>());
  if (invert && stream_rows) launch(invert_flags_kernel, grid_for(stream_rows, 256), 256, 0, stream(), flags.c->data.as<int8_t>(), stream_rows);
  return flags.release();
}

static JoinTable* jt_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null hash table handle");
  return reinterpret_cast<JoinTable*>((intptr_t)h);
}
static JoinTracker* tracker_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null join tracker handle");
  return reinterpret_cast<JoinTracker*>((intptr_t)h);
}

// GpuFilter directly below the stream side of an INNER FK -> PK join, fused INTO the probe (join_filter_probe_kernel) when
// the predicate is of the simple shape (simplefilter.cuh) and the probe qualifies for the one-key distinct probe: the gather
// maps carry ORIGINAL row ids of `batch`, `npass_out` = rows that passed the filter (the filter node's numOutputRows).
// tracker != 0: the build rows found are marked in it (join_filter_probe_kernel's tracking variant).
// false = not applicable, the caller takes the selection-vector path (b2_filter_row_ids + b2_join_probe_sel).
// whether join_filter_probe_kernel can probe `batch` with `prog` below it: the key column in `pc`, the predicate in `sp`
static bool filter_probe_applies(const JoinTable* jt, const Table* batch, int key_col, const Program* prog, const Column*& pc, SimplePred& sp) {
  if (getenv("B2_JOIN_NO_FAST_PROBE")) return false;
  const int64_t n = batch->rows;
  if (!jt->distinct || !jt->fast || jt->key_idx.size() != 1 || n < (1 << 16) || n >= 0x7fffffffLL) return false;
  if (key_col < 0 || key_col >= (int)batch->cols.size()) throw Error(B2_ERR_INVALID, "join key index out of range");
  pc = batch->cols[key_col];
  const int pw = dtype_width(pc->dtype);
  if (pc->nullable() || is_float(pc->dtype) || pc->dtype == B2_STRING || !(pw == 4 || pw == 8)) return false;
  if (pc->dtype != jt->keys->cols[jt->key_idx[0]]->dtype) return false;
  return simple_pred_of(prog, batch, sp);   // also: every predicate column 16-byte aligned
}

bool join_probe_pred(b2_handle ht, const Table* batch, int key_col, const Program* prog, Column** out_lm, Column** out_rm, int64_t* npass_out,
                     b2_handle tracker) {
  JoinTable* jt = jt_from(ht);
  uint32_t* track = nullptr;
  if (tracker) {
    JoinTracker* tr = tracker_from(tracker);
    if (tr->table != jt) throw Error(B2_ERR_INVALID, "join tracker belongs to another hash table");
    track = tr->bits.as<uint32_t>();
  }
  const int64_t n = batch->rows;
  const Column* pc = nullptr;
  SimplePred sp;
  if (!filter_probe_applies(jt, batch, key_col, prog, pc, sp)) return false;
  const int pw = dtype_width(pc->dtype);
  ColGuard lm(new_column(B2_INT32, 0, n, false)), rm(new_column(B2_INT32, 0, n, false));
  DevBuf tot(16);
  CUDA_CHECK(cudaMemsetAsync(tot.p, 0, 16, stream()));
  {
    const int grid = grid_for(n, FP_TILE, FP_CTAS);
    const uint64_t* sl = jt->slots.as<uint64_t>(); const uint32_t msk = (uint32_t)(jt->cap - 1);
    const unsigned long long* bl = jt->bloom.as<unsigned long long>();
    unsigned long long* tp = tot.as<unsigned long long>();
    int32_t* lp = lm.c->data.as<int32_t>(); int32_t* rp = rm.c->data.as<int32_t>();
    const NoEmit ne;
    if (track) {
      if (pw == 8) launch("join_filter_probe_track_kernel", join_filter_probe_kernel<int64_t, true>, grid, SF_NT, 0, stream(), sp, pc->data.as<int64_t>(), n,
                          sl, msk, bl, jt->bloom_mask, tp, lp, rp, tp + 1, track, ne);
      else launch("join_filter_probe_track_kernel", join_filter_probe_kernel<int32_t, true>, grid, SF_NT, 0, stream(), sp, pc->data.as<int32_t>(), n, sl,
                  msk, bl, jt->bloom_mask, tp, lp, rp, tp + 1, track, ne);
    } else if (pw == 8) {
      launch("join_filter_probe_kernel", join_filter_probe_kernel<int64_t, false>, grid, SF_NT, 0, stream(), sp, pc->data.as<int64_t>(), n, sl, msk, bl,
             jt->bloom_mask, tp, lp, rp, tp + 1, nullptr, ne);
    } else {
      launch("join_filter_probe_kernel", join_filter_probe_kernel<int32_t, false>, grid, SF_NT, 0, stream(), sp, pc->data.as<int32_t>(), n, sl, msk, bl,
             jt->bloom_mask, tp, lp, rp, tp + 1, nullptr, ne);
    }
  }
  unsigned long long h[2] = {0, 0};
  d2h(h, tot.p, 2);
  sync();
  lm.c->size = (int64_t)h[0]; rm.c->size = (int64_t)h[0];
  *npass_out = (int64_t)h[1];
  *out_lm = lm.release(); *out_rm = rm.release();
  return true;
}

// ---- the emitting probe's build payload: the build columns packed row-major, widest first so that every column sits at an
// offset that is a multiple of its width and none crosses an 8-byte word (a 16-byte column fills the row) -------------------
struct PackCols {
  int32_t n, words;
  int8_t w[EM_BUILD], off[EM_BUILD];
  const void* in[EM_BUILD];
};
__global__ void __launch_bounds__(256) join_pack_payload_kernel(const __grid_constant__ PackCols pc, int64_t rows, unsigned long long* __restrict__ out) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t lo = 0, hi = 0;
    for (int c = 0; c < pc.n; c++) {
      if (pc.w[c] == 16) { const ulonglong2 v = reinterpret_cast<const ulonglong2*>(pc.in[c])[r]; lo = v.x; hi = v.y; continue; }
      const uint64_t v = (pc.w[c] == 8 ? reinterpret_cast<const unsigned long long*>(pc.in[c])[r] : (uint64_t)reinterpret_cast<const uint32_t*>(pc.in[c])[r])
                         << (8 * (pc.off[c] & 7));
      if (pc.off[c] & 8) hi |= v; else lo |= v;
    }
    if (pc.words == 2) reinterpret_cast<ulonglong2*>(out)[r] = make_ulonglong2(lo, hi);
    else out[r] = lo;
  }
}

bool join_pack_payload(const Table* build, const std::vector<int>& cols, JoinPayload& pl) {
  if (cols.size() > (size_t)EM_BUILD) return false;
  int bytes = 0;
  for (int c : cols) {
    if (c < 0 || c >= (int)build->cols.size()) throw Error(B2_ERR_INVALID, "join column index out of range");
    const Column* bc = build->cols[c];
    if (bc->nullable() || bc->dtype == B2_STRING || !emit_width_ok(dtype_width(bc->dtype), true)) return false;
    bytes += dtype_width(bc->dtype);
  }
  if (bytes > 16) return false;
  pl.width = bytes == 0 ? 0 : (bytes <= 8 ? 8 : 16);
  pl.dtype.clear(); pl.scale.clear(); pl.off.assign(cols.size(), 0);
  for (int c : cols) { pl.dtype.push_back(build->cols[c]->dtype); pl.scale.push_back(build->cols[c]->scale); }
  PackCols pc; memset(&pc, 0, sizeof(pc));
  pc.words = pl.width / 8;
  int at = 0;
  for (int w = 16; w >= 4; w >>= 1)
    for (size_t k = 0; k < cols.size(); k++) {
      if (dtype_width(pl.dtype[k]) != w) continue;
      pl.off[k] = at;
      pc.w[pc.n] = (int8_t)w; pc.off[pc.n] = (int8_t)at; pc.in[pc.n] = build->cols[cols[k]]->data.p; pc.n++;
      at += w;
    }
  const int64_t rows = build->rows;
  pl.packed = DevBuf(pl.width ? (size_t)rows * pl.width : 0);
  if (pl.width && rows)
    launch("join_pack_payload_kernel", join_pack_payload_kernel, grid_for(rows, 256), 256, 0, stream(), pc, rows, pl.packed.as<unsigned long long>());
  return true;
}

bool join_probe_pred_emit(b2_handle ht, const Table* batch, int key_col, const Program* prog, const std::vector<int>& stream_cols,
                          const JoinPayload& pl, int64_t cap, Table** out, int64_t* total_out, int64_t* npass_out) {
  JoinTable* jt = jt_from(ht);
  const Column* pc = nullptr;
  SimplePred sp;
  if (!filter_probe_applies(jt, batch, key_col, prog, pc, sp) || stream_cols.size() > (size_t)EM_STREAM) return false;
  if (pl.packed.bytes != (size_t)jt->build_rows * pl.width) throw Error(B2_ERR_INVALID, "join payload does not match the hash table");
  for (int c : stream_cols) {
    if (c < 0 || c >= (int)batch->cols.size()) throw Error(B2_ERR_INVALID, "join column index out of range");
    const Column* ic = batch->cols[c];
    if (ic->nullable() || ic->dtype == B2_STRING || !emit_width_ok(dtype_width(ic->dtype), false)) return false;
  }
  EmitCols em; memset(&em, 0, sizeof(em));
  ColsGuard outs;
  for (int c : stream_cols) {
    const Column* ic = batch->cols[c];
    outs.v.push_back(new_column(ic->dtype, ic->scale, cap, false));
    em.s_w[em.ns] = (int8_t)dtype_width(ic->dtype);
    em.s_in[em.ns] = c == key_col ? nullptr : ic->data.p;
    em.s_out[em.ns++] = outs.v.back()->data.p;
  }
  for (size_t k = 0; k < pl.dtype.size(); k++) {
    outs.v.push_back(new_column(pl.dtype[k], pl.scale[k], cap, false));
    em.b_w[em.nb] = (int8_t)dtype_width(pl.dtype[k]); em.b_off[em.nb] = (int8_t)pl.off[k];
    em.b_out[em.nb++] = outs.v.back()->data.p;
  }
  em.pw = pl.width; em.packed = pl.packed.p; em.cap = (unsigned long long)cap;
  const int64_t n = batch->rows;
  DevBuf tot(16);
  CUDA_CHECK(cudaMemsetAsync(tot.p, 0, 16, stream()));
  {
    const int grid = grid_for(n, FP_TILE, FP_CTAS);
    const uint64_t* sl = jt->slots.as<uint64_t>(); const uint32_t msk = (uint32_t)(jt->cap - 1);
    const unsigned long long* bl = jt->bloom.as<unsigned long long>();
    unsigned long long* tp = tot.as<unsigned long long>();
    if (dtype_width(pc->dtype) == 8)
      launch("join_filter_probe_kernel", join_filter_probe_kernel<int64_t, false, true>, grid, SF_NT, 0, stream(), sp, pc->data.as<int64_t>(), n, sl, msk,
             bl, jt->bloom_mask, tp, nullptr, nullptr, tp + 1, nullptr, em);
    else
      launch("join_filter_probe_kernel", join_filter_probe_kernel<int32_t, false, true>, grid, SF_NT, 0, stream(), sp, pc->data.as<int32_t>(), n, sl, msk,
             bl, jt->bloom_mask, tp, nullptr, nullptr, tp + 1, nullptr, em);
  }
  unsigned long long h[2] = {0, 0};
  d2h(h, tot.p, 2);
  sync();
  *total_out = (int64_t)h[0];
  *npass_out = (int64_t)h[1];
  if ((int64_t)h[0] <= cap) {
    for (Column* c : outs.v) c->size = (int64_t)h[0];
    *out = new_table(outs.release());
  }
  return true;
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_join_build(b2_handle build_keys_table, int32_t nulls_equal, b2_handle* out_hash_table) {
  B2_TRY
  Table* t = table_from(build_keys_table);
  B2_CHECK(!t->cols.empty() && (int)t->cols.size() <= MAX_KEYS, "join needs 1..8 key columns");
  std::unique_ptr<JoinTable> jt(new JoinTable());
  t->refs.fetch_add(1);
  jt->keys = t;
  jt->build_rows = t->rows;
  jt->nulls_equal = nulls_equal != 0;
  for (int i = 0; i < (int)t->cols.size(); i++) jt->key_idx.push_back(i);
  int64_t cap = 1024;
  while (cap < t->rows * 2) cap <<= 1;
  jt->cap = cap;
  {
    int kw = 0; bool fixed = true, nullable = false;
    for (auto* c : t->cols) { if (c->dtype == B2_STRING || c->dtype == B2_DECIMAL128) fixed = false; kw += dtype_width(c->dtype); nullable = nullable || c->nullable(); }
    jt->fast = fixed && kw <= 8 && !(jt->nulls_equal && nullable);
  }
  jt->slots = DevBuf((size_t)cap * (jt->fast ? 16 : 8));
  CUDA_CHECK(cudaMemsetAsync(jt->slots.p, 0xff, jt->slots.bytes, stream()));
  if (t->rows >= (1 << 18) && !getenv("B2_JOIN_NO_BLOOM")) {   // smaller tables are L2 resident themselves
    // bits per key: fewer bits = more false positives (each costs one random HBM slot read) but a smaller filter.  SF100 q3
    // step on one H100 SXM (700 W): 8 bits 37.6 ms (probe 8.8), 16 bits 40.6 ms (probe 11.3): the 32 MB filter of the
    // 14.6 M-row build side crowds the 50 MB L2, the 16 MB one does not.  Pinning the 16-bit filter in the persisting part
    // of L2 (B2_JOIN_BLOOM_PERSIST) was slower still (55.5 ms)
    static const int bits_per_key = getenv("B2_JOIN_BLOOM_BITS") ? std::max(2, atoi(getenv("B2_JOIN_BLOOM_BITS"))) : 8;
    int64_t words = 1 << 15;
    while (words * 64 < t->rows * bits_per_key && words < (4 << 20)) words <<= 1;   // at most 32 MB
    if (words * 64 >= t->rows * 6) {                                // below ~6 bits per key the filter stops paying
      jt->bloom = DevBuf((size_t)words * 8);
      // bits set per key, same step at 8 bits/key: k=2 38.2 ms, k=3 37.4 / 37.3, k=4 36.9 / 37.3 (within noise of k=3)
      static const int bloom_k = getenv("B2_JOIN_BLOOM_K") ? std::min(4, std::max(2, atoi(getenv("B2_JOIN_BLOOM_K")))) : 3;
      jt->bloom_mask = (uint32_t)(words - 1) | ((uint32_t)(bloom_k - 2) << 28);
      CUDA_CHECK(cudaMemsetAsync(jt->bloom.p, 0, jt->bloom.bytes, stream()));
    }
  }
  DevBuf dups(4);
  CUDA_CHECK(cudaMemsetAsync(dups.p, 0, 4, stream()));
  if (t->rows) {
    KeyCols keys = key_cols_of(t, jt->key_idx.data(), (int)jt->key_idx.size());
    launch("join_build_kernel", join_build_kernel, grid_for(t->rows, 256), 256, 0, stream(), keys, t->rows, jt->slots.as<uint64_t>(), (uint32_t)(cap - 1),
           jt->nulls_equal, jt->fast, dups.as<int32_t>(), jt->bloom.as<unsigned long long>(), jt->bloom_mask);
  }
  int32_t h_dups = 0;
  d2h(&h_dups, dups.p, 1);
  sync();
  jt->distinct = h_dups == 0;
  *out_hash_table = to_handle(jt.release());
  B2_CATCH
}

int b2_join_hash_table_close(b2_handle ht) {
  B2_TRY
  delete jt_from(ht);
  B2_CATCH
}

int b2_join_probe_filter(b2_handle ht, b2_handle table, int32_t key_col, b2_handle predicate_program, b2_handle* out_left_map,
                         b2_handle* out_right_map, int64_t* out_npass) {
  B2_TRY
  Table* t = table_from(table);
  B2_CHECK(key_col >= 0 && key_col < (int)t->cols.size(), "join key index out of range");
  Column* lm = nullptr; Column* rm = nullptr;
  int64_t npass = 0;
  if (join_probe_pred(ht, t, key_col, program_from(predicate_program), &lm, &rm, &npass, 0)) {
    *out_left_map = to_handle(lm); *out_right_map = to_handle(rm); *out_npass = npass;
    return B2_OK;
  }
  b2_handle sel = 0;
  int rc = b2_filter_row_ids(predicate_program, table, &sel);
  if (rc != B2_OK) return rc;
  ColGuard sg(col_from(sel));
  col_incref(t->cols[key_col]);
  std::unique_ptr<Table, void (*)(Table*)> keys(new_table({t->cols[key_col]}), table_release);
  rc = b2_join_probe_sel(ht, to_handle(keys.get()), sel, B2_JOIN_INNER, out_left_map, out_right_map);
  if (rc != B2_OK) return rc;
  *out_npass = sg.c->size;
  B2_CATCH
}

int b2_join_probe(b2_handle ht, b2_handle probe_keys_table, int32_t kind, b2_handle* out_left_map, b2_handle* out_right_map) {
  return b2_join_probe_sel(ht, probe_keys_table, 0, kind, out_left_map, out_right_map);
}

}  // extern "C"

namespace b2 {
// The probe proper: kinds INNER .. LEFT_ANTI, through an optional selection vector; track != nullptr (INNER / LEFT OUTER only)
// takes the tracking variant of whichever probe kernel runs.
static void probe_maps(JoinTable* jt, Table* pt, b2_handle selection, int32_t kind, uint32_t* track, b2_handle* out_left_map, b2_handle* out_right_map) {
  const int32_t* sel = nullptr;
  int64_t nsel = 0;
  if (selection) {
    Column* sc = col_from(selection);
    B2_CHECK(sc->dtype == B2_INT32, "selection vector must be INT32");
    sel = sc->data.as<int32_t>(); nsel = sc->size;
  }
  B2_CHECK(pt->cols.size() == jt->keys->cols.size(), "probe and build key counts differ");
  for (size_t i = 0; i < pt->cols.size(); i++)
    B2_CHECK(pt->cols[i]->dtype == jt->keys->cols[i]->dtype, "probe and build key dtypes differ");
  B2_CHECK(kind >= B2_JOIN_INNER && kind <= B2_JOIN_LEFT_ANTI, "bad join kind");
  // an empty selection vector has no data buffer (sel == nullptr) and selects no row
  const int64_t n = selection ? nsel : pt->rows;
  const bool semi_like = kind == B2_JOIN_LEFT_SEMI || kind == B2_JOIN_LEFT_ANTI;
  KeyCols pk = key_cols_of(pt, jt->key_idx.data(), (int)jt->key_idx.size());
  KeyCols bk = key_cols_of(jt->keys, jt->key_idx.data(), (int)jt->key_idx.size());
  if (jt->distinct && (kind == B2_JOIN_INNER || kind == B2_JOIN_LEFT_OUTER)) {
    // innerDistinctJoinGatherMaps / leftDistinctJoinGatherMap fast path (GpuHashJoin.scala:1401-1428)
    ColGuard lm(new_column(B2_INT32, 0, n, false)), rm(new_column(B2_INT32, 0, n, false));
    int64_t matched = n;
    if (n) {
      DevBuf tot(8);
      CUDA_CHECK(cudaMemsetAsync(tot.p, 0, 8, stream()));
      L2Persist keep(jt->bloom.p, jt->bloom.bytes);
      const Column* pc = jt->key_idx.size() == 1 ? pt->cols[jt->key_idx[0]] : nullptr;
      const int pw = pc ? dtype_width(pc->dtype) : 0;
      if (kind == B2_JOIN_INNER && jt->fast && pc && !pc->nullable() && !is_float(pc->dtype) && pc->dtype != B2_STRING && (pw == 4 || pw == 8) &&
          n < 0x7fffffffLL && !getenv("B2_JOIN_NO_FAST_PROBE")) {
        const int grid = grid_for(n, 256);
        const uint64_t* sl = jt->slots.as<uint64_t>(); const uint32_t msk = (uint32_t)(jt->cap - 1);
        const unsigned long long* bl = jt->bloom.as<unsigned long long>(); unsigned long long* tp = tot.as<unsigned long long>();
        int32_t* lp = lm.c->data.as<int32_t>(); int32_t* rp = rm.c->data.as<int32_t>();
        if (track) {
          if (pw == 8)
            launch("join_probe_distinct1_track_kernel", sel ? join_probe_distinct1_kernel<int64_t, true, true> : join_probe_distinct1_kernel<int64_t, false, true>,
                   grid, 256, 0, stream(), pc->data.as<int64_t>(), sel, n, sl, msk, bl, jt->bloom_mask, tp, lp, rp, track);
          else
            launch("join_probe_distinct1_track_kernel", sel ? join_probe_distinct1_kernel<int32_t, true, true> : join_probe_distinct1_kernel<int32_t, false, true>,
                   grid, 256, 0, stream(), pc->data.as<int32_t>(), sel, n, sl, msk, bl, jt->bloom_mask, tp, lp, rp, track);
        } else if (pw == 8) {
          launch("join_probe_distinct1_kernel", sel ? join_probe_distinct1_kernel<int64_t, true, false> : join_probe_distinct1_kernel<int64_t, false, false>,
                 grid, 256, 0, stream(), pc->data.as<int64_t>(), sel, n, sl, msk, bl, jt->bloom_mask, tp, lp, rp, nullptr);
        } else {
          launch("join_probe_distinct1_kernel", sel ? join_probe_distinct1_kernel<int32_t, true, false> : join_probe_distinct1_kernel<int32_t, false, false>,
                 grid, 256, 0, stream(), pc->data.as<int32_t>(), sel, n, sl, msk, bl, jt->bloom_mask, tp, lp, rp, nullptr);
        }
      } else {
        launch(track ? "join_probe_distinct_track_kernel" : "join_probe_distinct_kernel",
               track ? join_probe_distinct_kernel<true> : join_probe_distinct_kernel<false>, grid_for(n, 256), 256, 0, stream(), pk, bk, n,
               jt->slots.as<uint64_t>(), (uint32_t)(jt->cap - 1), jt->nulls_equal, jt->fast, kind, tot.as<unsigned long long>(), lm.c->data.as<int32_t>(),
               rm.c->data.as<int32_t>(), jt->bloom.as<unsigned long long>(), jt->bloom_mask, sel, track);
      }
      if (kind == B2_JOIN_INNER) { unsigned long long h = 0; d2h(&h, tot.p, 1); sync(); matched = (int64_t)h; }
    }
    lm.c->size = matched; rm.c->size = matched;  // buffers stay sized for n rows
    *out_left_map = to_handle(lm.release());
    if (out_right_map) *out_right_map = to_handle(rm.release()); else col_release(rm.release());
    return;
  }
  DevBuf counts((size_t)std::max<int64_t>(n, 1) * 4), offsets((size_t)(n + 1) * 8);
  int64_t total = 0;
  if (n) {
    launch("join_probe_count_kernel", join_probe_kernel<0>, grid_for(n, 256), 256, 0, stream(), pk, bk, n, jt->slots.as<uint64_t>(), (uint32_t)(jt->cap - 1),
           jt->nulls_equal, jt->fast, kind, counts.as<int32_t>(), nullptr, nullptr, nullptr, jt->bloom.as<unsigned long long>(), jt->bloom_mask, sel, nullptr);
    exclusive_scan<int32_t, int64_t>(counts.as<int32_t>(), offsets.as<int64_t>(), n, true);
    d2h(&total, offsets.as<int64_t>() + n, 1);
    sync();
  }
  // the reference splits the stream batch when the maps would pass the batch target
  // (AbstractGpuJoinIterator.scala:235-250); the hard limit here is the int32 row index
  if (total > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "join output exceeds 2^31-1 rows; split the stream batch");
  ColGuard lm(new_column(B2_INT32, 0, total, false));
  ColGuard rm(semi_like ? nullptr : new_column(B2_INT32, 0, total, false));
  if (n && total)
    launch(track ? "join_probe_write_track_kernel" : "join_probe_write_kernel", track ? join_probe_kernel<1, true> : join_probe_kernel<1, false>,
           grid_for(n, 256), 256, 0, stream(), pk, bk, n, jt->slots.as<uint64_t>(), (uint32_t)(jt->cap - 1), jt->nulls_equal, jt->fast, kind, nullptr,
           offsets.as<int64_t>(), lm.c->data.as<int32_t>(), semi_like ? nullptr : rm.c->data.as<int32_t>(), jt->bloom.as<unsigned long long>(),
           jt->bloom_mask, sel, track);
  *out_left_map = to_handle(lm.release());
  if (out_right_map) *out_right_map = semi_like ? 0 : to_handle(rm.release());
}

// maps (lo, ro) of m rows, then (INT32_MIN, b) for every build row b whose bit is clear in `tr`, ascending
static void append_unmatched(const JoinTracker* tr, const Column* lo, const Column* ro, b2_handle* out_left_map, b2_handle* out_right_map) {
  const int64_t m = lo->size;
  DevBuf offs;
  const int64_t extra = tracker_unmatched_count(tr, offs);
  if (m + extra > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "join output exceeds 2^31-1 rows; split the stream batch");
  ColGuard lm(new_column(B2_INT32, 0, m + extra, false)), rm(new_column(B2_INT32, 0, m + extra, false));
  if (m) {
    CUDA_CHECK(cudaMemcpyAsync(lm.c->data.p, lo->data.p, (size_t)m * 4, cudaMemcpyDeviceToDevice, stream()));
    CUDA_CHECK(cudaMemcpyAsync(rm.c->data.p, ro->data.p, (size_t)m * 4, cudaMemcpyDeviceToDevice, stream()));
  }
  tracker_unmatched_write(tr, offs, extra, rm.c->data.as<int32_t>() + m, lm.c->data.as<int32_t>() + m);
  *out_left_map = to_handle(lm.release());
  *out_right_map = to_handle(rm.release());
}
}  // namespace b2

extern "C" {

// probe through a selection vector: `selection` (INT32 row ids into probe_keys_table, ascending, e.g. from b2_filter_row_ids)
// names the stream rows that take part; the left gather map carries ORIGINAL row ids of probe_keys_table's batch
int b2_join_probe_sel(b2_handle ht, b2_handle probe_keys_table, b2_handle selection, int32_t kind, b2_handle* out_left_map, b2_handle* out_right_map) {
  B2_TRY
  JoinTable* jt = jt_from(ht);
  Table* pt = table_from(probe_keys_table);
  if (kind == B2_JOIN_FULL_OUTER || kind == B2_JOIN_RIGHT_OUTER) {
    // FULL OUTER: the left outer maps; RIGHT OUTER: the inner maps (marking the build rows found as it goes).  Then one extra
    // row (left = out of bounds -> NULLs) per build row that nothing matched, ascending
    B2_CHECK(out_right_map != nullptr, "an outer join that preserves the build side needs both gather maps");
    B2_CHECK(!(selection && kind == B2_JOIN_FULL_OUTER), "full outer join through a selection vector");
    std::unique_ptr<JoinTracker> tr(tracker_new(jt, jt->keys->rows));
    b2_handle hl = 0, hr = 0;
    if (kind == B2_JOIN_FULL_OUTER) probe_maps(jt, pt, 0, B2_JOIN_LEFT_OUTER, nullptr, &hl, &hr);
    else probe_maps(jt, pt, selection, B2_JOIN_INNER, tr->bits.as<uint32_t>(), &hl, &hr);
    ColGuard lo(col_from(hl)), ro(col_from(hr));
    if (kind == B2_JOIN_FULL_OUTER) tracker_mark(tr.get(), ro.c->data.as<int32_t>(), ro.c->size, nullptr);
    append_unmatched(tr.get(), lo.c, ro.c, out_left_map, out_right_map);
    return B2_OK;
  }
  probe_maps(jt, pt, selection, kind, nullptr, out_left_map, out_right_map);
  B2_CATCH
}

int b2_join_tracker_create(b2_handle ht, b2_handle* out_tracker) {
  B2_TRY
  JoinTable* jt = jt_from(ht);
  *out_tracker = to_handle(tracker_new(jt, jt->build_rows));
  B2_CATCH
}

int b2_join_tracker_close(b2_handle tracker) {
  B2_TRY
  delete tracker_from(tracker);
  B2_CATCH
}

int b2_join_probe_track(b2_handle ht, b2_handle probe_keys_table, b2_handle selection, int32_t kind, b2_handle tracker, b2_handle* out_left_map,
                        b2_handle* out_right_map) {
  B2_TRY
  JoinTable* jt = jt_from(ht);
  JoinTracker* tr = tracker_from(tracker);
  B2_CHECK(tr->table == jt, "join tracker belongs to another hash table");
  B2_CHECK(kind == B2_JOIN_INNER || kind == B2_JOIN_LEFT_OUTER, "only inner and left outer probes write the maps a tracker follows");
  B2_CHECK(out_right_map != nullptr, "a tracked probe needs both gather maps");
  probe_maps(jt, table_from(probe_keys_table), selection, kind, tr->bits.as<uint32_t>(), out_left_map, out_right_map);
  B2_CATCH
}

int b2_join_tracker_mark(b2_handle tracker, b2_handle right_map, b2_handle pass) {
  B2_TRY
  JoinTracker* tr = tracker_from(tracker);
  const Column* rm = col_from(right_map);
  B2_CHECK(rm->dtype == B2_INT32, "right gather map must be INT32");
  const Column* pc = pass ? col_from(pass) : nullptr;
  B2_CHECK(!pc || (pc->dtype == B2_BOOL8 && pc->size == rm->size), "pass mask must be BOOL8 with one row per map entry");
  tracker_mark(tr, rm->data.as<int32_t>(), rm->size, pc);
  int32_t bad = 0;
  d2h(&bad, tr->bad.p, 1);
  sync();
  if (bad) {
    CUDA_CHECK(cudaMemsetAsync(tr->bad.p, 0, 4, stream()));
    throw Error(B2_ERR_INVALID, "right gather map entry past the build side");
  }
  B2_CATCH
}

int b2_join_tracker_unmatched(b2_handle tracker, b2_handle* out_ids) {
  B2_TRY
  const JoinTracker* tr = tracker_from(tracker);
  DevBuf offs;
  const int64_t u = tracker_unmatched_count(tr, offs);
  ColGuard ids(new_column(B2_INT32, 0, u, false));
  tracker_unmatched_write(tr, offs, u, ids.c->data.as<int32_t>(), nullptr);
  *out_ids = to_handle(ids.release());
  B2_CATCH
}

}  // extern "C"
