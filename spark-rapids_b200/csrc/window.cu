// window.cu — a13: window functions over a batch sorted by (partition keys, order keys).
// Reference: GpuWindowExec.scala:32-52, 145-161; GpuRunningWindowExec.scala:42-250; GpuWindowExpression.scala:531 (frames),
// :843 (BatchedRunningWindowFixer), :1367-1600 (SumBinaryFixer), :1645, :1772 (RankFixer, DenseRankFixer), :1912-2110 (rank,
// dense_rank, row_number, lead, lag); BasicWindowCalc.scala:435-521 (the cudf aggregateWindows / scan / groupBy.scan calls).
//
// Kernels:
//   window_bounds_kernel      partition and peer starts, from the sort's normalised key bytes (sortkey.cuh); row 0 is compared
//                             with the previous chunk's last row when one is carried
//   window_scan_kernel        segmented inclusive scan (restarting at partition starts) of one function's state, single pass
//                             with decoupled look-back; the look-back stops at the first predecessor tile with a partition start.
//                             Payloads wider than 64 bits are published beside a status word, written after a fence.  The
//                             batch carry-in is the state before row 0; the last tile writes the carry-out.
//   window_group_ends_kernel  last row of each partition / peer group, stored at the group's first row
//   window_finish_kernel      each row's frame [s, e] clipped to its partition, evaluated from the scan state: the state at e when
//                             s is the partition start (running, RANGE running = e at the peer group's end, whole partition = e
//                             at the partition's end), a difference of prefixes for integer, decimal and count sums, otherwise a
//                             loop over the frame (float SUM, MIN, MAX: O(rows x frame width), as cudf's rolling window)
//   window_lead_lag_kernel    LEAD / LAG source row (or -1 outside the partition); values through gather_table, then the default
//   window_value_kernel       FIRST / LAST / NTH_VALUE source row of each row's frame (or -1: NULL, or n: the carried value), with
//                             IGNORE NULLS a select on a rank directory of the validity words (window_valid_popc_kernel + a
//                             scan); values through gather_table, then window_value_patch_kernel writes the carried value.
//                             window_value_carry_kernel takes the next carry (count and source row) at the carry row
// Finish, LEAD / LAG and the value functions run over every row of the chunk (AllRows) or, for a streamed bounded plan, only over the rows [lo, hi)
// between its context and look-ahead rows (RowRange), writing columns of hi - lo rows.
// RANGE frames with value offsets (B2_FRAME_RANGE_VALUE; BasicWindowCalc.scala:169-219, 445 aggregateWindowsOverRanges):
//   window_range_bounds_kernel  each row's frame [s, e], once per distinct (lower, upper): a binary search of the ORDER BY
//                               values in the partition for a value offset, the peer-group or partition edge otherwise
//   window_range_tiles_kernel   non-SUB ops (float SUM, MIN, MAX): per WIN_TILE-row tile the unsegmented in-tile prefix and
//                               suffix of the state and the tile's aggregate
//   window_range_table_kernel   one level of a sparse table over the tile aggregates (level k: tiles [t, t + 2^k))
//   window_range_finish_kernel  the frame's value: state[e] from the partition start, a difference of prefixes for SUB ops,
//                               otherwise suffix[s] + O(log tiles) levels + prefix[e] (a loop when s and e share a tile), so
//                               the work per row is bounded by WIN_TILE + log2(tiles) whatever the frame's width
#include <algorithm>
#include "prim.cuh"
#include "sortkey.cuh"
#include "window.cuh"

namespace b2 {

Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols);
Table* slice_table(const Table* t, int64_t start, int64_t end);
Table* concat_tables(const std::vector<const Table*>& ts);

constexpr int WIN_NT = 128, WIN_ITEMS = 8, WIN_TILE = WIN_NT * WIN_ITEMS;   // 1024 rows per scan tile
constexpr uint8_t F_PART = 1, F_PEER = 2;                                      // a partition start is also a peer start

// ------------------------------------------------------------------------------------------------
// boundaries
__device__ __forceinline__ bool keys_equal(const SortPlan& a, int64_t ra, const SortPlan& b, int64_t rb) {
  for (int ci = 0; ci < a.ncols; ci++)
    for (int k = 0; k < a.c[ci].key_len; k++)
      if (norm_byte(a.c[ci], ra, k) != norm_byte(b.c[ci], rb, k)) return false;
  return true;
}

__global__ void window_bounds_kernel(const __grid_constant__ SortPlan part, const __grid_constant__ SortPlan order,
                                     const __grid_constant__ SortPlan cpart, const __grid_constant__ SortPlan corder, int has_carry, int64_t n,
                                     uint8_t* __restrict__ flags) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool ps, qs;
    if (i == 0 && !has_carry) ps = qs = true;
    else if (i == 0) { ps = !keys_equal(part, 0, cpart, 0); qs = ps || !keys_equal(order, 0, corder, 0); }
    else { ps = !keys_equal(part, i, part, i - 1); qs = ps || !keys_equal(order, i, order, i - 1); }
    flags[i] = (ps ? F_PART : 0) | (qs ? F_PEER : 0);
  }
}

// the last row (or -1) whose flags have a bit of `mask`
__global__ void window_last_start_kernel(const uint8_t* __restrict__ flags, int64_t n, uint8_t mask, unsigned long long* out) {
  long long best = -1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (flags[i] & mask) best = i;
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best >= 0) atomicMax(reinterpret_cast<long long*>(out), best);
}

// ------------------------------------------------------------------------------------------------
// scan states
struct I192 { uint64_t w[3]; };
__device__ __forceinline__ I192 i192_of(i128 v) { I192 r; r.w[0] = (uint64_t)v; r.w[1] = (uint64_t)((u128)v >> 64); r.w[2] = v < 0 ? ~0ull : 0ull; return r; }
__device__ __forceinline__ I192 i192_add(const I192& a, const I192& b) {
  I192 r;
  r.w[0] = a.w[0] + b.w[0];
  const uint64_t c0 = r.w[0] < a.w[0];
  const uint64_t s1 = a.w[1] + b.w[1];
  const uint64_t c1 = s1 < a.w[1];
  r.w[1] = s1 + c0;
  const uint64_t c2 = c1 | (r.w[1] < s1);
  r.w[2] = a.w[2] + b.w[2] + c2;
  return r;
}
__device__ __forceinline__ I192 i192_neg(const I192& a) {
  I192 n{{~a.w[0], ~a.w[1], ~a.w[2]}};
  return i192_add(n, I192{{1, 0, 0}});
}
__device__ __forceinline__ bool i192_lt(const I192& a, const I192& b) {
  if (a.w[2] != b.w[2]) return (int64_t)a.w[2] < (int64_t)b.w[2];
  if (a.w[1] != b.w[1]) return a.w[1] < b.w[1];
  return a.w[0] < b.w[0];
}
// |v| < 10^p
__device__ __forceinline__ bool i192_fits(const I192& v, int p) {
  i128 lim = 1;
  for (int k = 0; k < p; k++) lim *= 10;
  return i192_lt(v, i192_of(lim)) && i192_lt(i192_of(-lim), v);
}

__device__ __forceinline__ int64_t load_int(const ColView& c, int64_t i) {
  switch (c.width) {
    case 1: return reinterpret_cast<const int8_t*>(c.data)[i];
    case 2: return reinterpret_cast<const int16_t*>(c.data)[i];
    case 4: return reinterpret_cast<const int32_t*>(c.data)[i];
    default: return reinterpret_cast<const int64_t*>(c.data)[i];
  }
}
__device__ __forceinline__ double load_float(const ColView& c, int64_t i) {
  return c.dtype == B2_FLOAT32 ? (double)reinterpret_cast<const float*>(c.data)[i] : reinterpret_cast<const double*>(c.data)[i];
}
// order-preserving u64 of a MIN/MAX input: b2_groupby's map (agg.cu ord_i64 / ord_f64: NaN greatest, -0.0 = 0.0)
__device__ __forceinline__ uint64_t ord_key(const ColView& c, int64_t i) {
  if (c.dtype == B2_FLOAT32 || c.dtype == B2_FLOAT64) {
    double d = load_float(c, i);
    if (d != d) return 0xffffffffffffffffull;
    if (d == 0.0) d = 0.0;
    const uint64_t b = (uint64_t)__double_as_longlong(d);
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
  }
  return (uint64_t)load_int(c, i) ^ 0x8000000000000000ull;
}

// the output of one function: values, validity (zeroed) and the result precision of decimal sums
struct WinOut {
  void* data;
  uint32_t* valid;
  int32_t dtype, precision;
  int32_t field;   // ranking: 0 row_number, 1 rank, 2 dense_rank
};
__device__ __forceinline__ void set_valid(const WinOut& o, int64_t i) { atomicOr(&o.valid[i >> 5], 1u << (i & 31)); }

// ROW_NUMBER / RANK / DENSE_RANK in one state: rows since the partition start, row number at the last peer start, peer starts
struct RankOp {
  struct T { int64_t rn, rk, dr, hp; };
  const uint8_t* flags;
  static constexpr bool SUB = false;
  __device__ T identity() const { return T{0, 0, 0, 0}; }
  __device__ T elem(int64_t i) const { const int64_t p = (flags[i] & F_PEER) ? 1 : 0; return T{1, p, p, p}; }
  __device__ T combine(const T& a, const T& b) const { return T{a.rn + b.rn, b.hp ? a.rn + b.rk : a.rk, a.dr + b.dr, a.hp | b.hp}; }
  __device__ T sub(const T& a, const T&) const { return a; }
  __device__ void finish(const T& v, bool, const WinOut& o, int64_t i) const {
    reinterpret_cast<int32_t*>(o.data)[i] = (int32_t)(o.field == 0 ? v.rn : o.field == 1 ? v.rk : v.dr);
    set_valid(o, i);
  }
};

struct CountOp {
  struct T { int64_t c; };
  ColView col;
  int all;
  static constexpr bool SUB = true;
  __device__ T identity() const { return T{0}; }
  __device__ T elem(int64_t i) const { return T{(all || row_valid(col.valid, i)) ? 1 : 0}; }
  __device__ T combine(const T& a, const T& b) const { return T{a.c + b.c}; }
  __device__ T sub(const T& a, const T& b) const { return T{a.c - b.c}; }
  __device__ void finish(const T& v, bool, const WinOut& o, int64_t i) const {
    reinterpret_cast<int64_t*>(o.data)[i] = v.c;
    set_valid(o, i);
  }
};

// integer SUM: wraps like Java's long (non-ANSI)
struct SumIntOp {
  struct T { uint64_t s; int64_t nv; };
  ColView col;
  static constexpr bool SUB = true;
  __device__ T identity() const { return T{0, 0}; }
  __device__ T elem(int64_t i) const { return row_valid(col.valid, i) ? T{(uint64_t)load_int(col, i), 1} : T{0, 0}; }
  __device__ T combine(const T& a, const T& b) const { return T{a.s + b.s, a.nv + b.nv}; }
  __device__ T sub(const T& a, const T& b) const { return T{a.s - b.s, a.nv - b.nv}; }
  __device__ void finish(const T& v, bool, const WinOut& o, int64_t i) const {
    reinterpret_cast<int64_t*>(o.data)[i] = (int64_t)v.s;
    if (v.nv > 0) set_valid(o, i);
  }
};

// float SUM in double; never a difference of prefixes (cancellation, inf - inf)
struct SumFloatOp {
  struct T { double s; int64_t nv; };
  ColView col;
  static constexpr bool SUB = false;
  __device__ T identity() const { return T{0.0, 0}; }
  // every sum starts from 0.0, as Spark's (coalesce(sum, 0) + x): a first value of -0.0 gives 0.0, also at a segment start
  __device__ T elem(int64_t i) const { return row_valid(col.valid, i) ? T{load_float(col, i) + 0.0, 1} : T{0.0, 0}; }
  __device__ T combine(const T& a, const T& b) const { return T{a.s + b.s, a.nv + b.nv}; }
  __device__ T sub(const T& a, const T&) const { return a; }
  __device__ void finish(const T& v, bool, const WinOut& o, int64_t i) const {
    reinterpret_cast<double*>(o.data)[i] = v.s;
    if (v.nv > 0) set_valid(o, i);
  }
};

// exact decimal SUM in 192 bits, with the largest and smallest running value of the piece: a running sum is NULL from the
// first row whose running value does not fit the result precision on (SumBinaryFixer), which is "the largest or the smallest
// running value so far does not fit".  A prefix of 0 is counted among the running values; it always fits, so it never matters.
struct SumDecOp {
  struct T { I192 s, mx, mn; int64_t nv; };
  ColView col;
  static constexpr bool SUB = true;
  __device__ T identity() const { const I192 z{{0, 0, 0}}; return T{z, z, z, 0}; }
  __device__ T elem(int64_t i) const {
    if (!row_valid(col.valid, i)) return identity();
    i128 v;
    if (col.width == 16) v = reinterpret_cast<const i128*>(col.data)[i];
    else v = (i128)load_int(col, i);
    const I192 x = i192_of(v), z{{0, 0, 0}};
    return T{x, i192_lt(z, x) ? x : z, i192_lt(x, z) ? x : z, 1};
  }
  __device__ T combine(const T& a, const T& b) const {
    const I192 hi = i192_add(a.s, b.mx), lo = i192_add(a.s, b.mn);
    return T{i192_add(a.s, b.s), i192_lt(a.mx, hi) ? hi : a.mx, i192_lt(lo, a.mn) ? lo : a.mn, a.nv + b.nv};
  }
  __device__ T sub(const T& a, const T& b) const { return T{i192_add(a.s, i192_neg(b.s)), a.mx, a.mn, a.nv - b.nv}; }
  __device__ void finish(const T& v, bool running, const WinOut& o, int64_t i) const {
    const bool ok = v.nv > 0 && (running ? (i192_fits(v.mx, o.precision) && i192_fits(v.mn, o.precision)) : i192_fits(v.s, o.precision));
    const i128 x = (i128)(((u128)v.s.w[1] << 64) | v.s.w[0]);
    if (o.dtype == B2_DECIMAL128) reinterpret_cast<i128*>(o.data)[i] = ok ? x : (i128)0;
    else reinterpret_cast<int64_t*>(o.data)[i] = ok ? (int64_t)x : 0;
    if (ok) set_valid(o, i);
  }
};

struct MinMaxOp {
  struct T { uint64_t k; int64_t nv; };
  ColView col;
  int is_max;
  static constexpr bool SUB = false;
  __device__ T identity() const { return T{is_max ? 0ull : ~0ull, 0}; }
  __device__ T elem(int64_t i) const { return row_valid(col.valid, i) ? T{ord_key(col, i), 1} : identity(); }
  __device__ T combine(const T& a, const T& b) const { return T{is_max ? max(a.k, b.k) : min(a.k, b.k), a.nv + b.nv}; }
  __device__ T sub(const T& a, const T&) const { return a; }
  __device__ void finish(const T& v, bool, const WinOut& o, int64_t i) const {
    if (v.nv == 0) { memset(reinterpret_cast<char*>(o.data) + i * col.width, 0, col.width); return; }
    if (col.dtype == B2_FLOAT32 || col.dtype == B2_FLOAT64) {
      double d;
      if (v.k == 0xffffffffffffffffull) d = __longlong_as_double(0x7ff8000000000000ll);
      else d = __longlong_as_double((long long)((v.k & 0x8000000000000000ull) ? (v.k & 0x7fffffffffffffffull) : ~v.k));
      if (col.dtype == B2_FLOAT32) reinterpret_cast<float*>(o.data)[i] = (float)d;
      else reinterpret_cast<double*>(o.data)[i] = d;
    } else {
      const int64_t x = (int64_t)(v.k ^ 0x8000000000000000ull);
      switch (col.width) {
        case 1: reinterpret_cast<int8_t*>(o.data)[i] = (int8_t)x; break;
        case 2: reinterpret_cast<int16_t*>(o.data)[i] = (int16_t)x; break;
        case 4: reinterpret_cast<int32_t*>(o.data)[i] = (int32_t)x; break;
        default: reinterpret_cast<int64_t*>(o.data)[i] = x; break;
      }
    }
    set_valid(o, i);
  }
};

// ------------------------------------------------------------------------------------------------
// segmented scan with decoupled look-back
template <typename T>
struct Seg { T v; uint64_t f; };   // f: the piece contains a partition start (what came before it does not count)

template <class Op, typename S>
__device__ __forceinline__ S seg_combine(const Op& op, const S& a, const S& b) {
  if (b.f) return b;
  return S{op.combine(a.v, b.v), a.f};
}
// a published tile payload, read past L1
template <typename S>
__device__ __forceinline__ S ld_cg(const S* p) {
  static_assert(sizeof(S) % 8 == 0, "payloads are whole 8-byte words");
  S r;
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(p);
  unsigned long long* d = reinterpret_cast<unsigned long long*>(&r);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(S) / 8); k++) d[k] = __ldcg(s + k);
  return r;
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v) { asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

constexpr uint32_t TS_AGG = 1, TS_PREFIX = 2;

// state[i] = the function's state over rows [partition start, i]; carry_in (may be null) = the state before row 0
template <class Op>
__global__ void __launch_bounds__(WIN_NT) window_scan_kernel(const Op op, const uint8_t* __restrict__ flags, int64_t n,
                                                             typename Op::T* __restrict__ state, const typename Op::T* carry_in,
                                                             typename Op::T* carry_out, unsigned long long* tile_counter, uint32_t* status,
                                                             Seg<typename Op::T>* t_agg, Seg<typename Op::T>* t_inc) {
  using S = Seg<typename Op::T>;
  __shared__ S s_scan[2][WIN_NT];
  __shared__ S s_excl;
  __shared__ int64_t s_tile;
  const int64_t ntiles = (n + WIN_TILE - 1) / WIN_TILE;
  while (true) {
    // tiles are claimed in launch order, so a look-back only waits on tiles whose CTAs are running
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(tile_counter, 1ull);
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    const int64_t base = tile * WIN_TILE + (int64_t)threadIdx.x * WIN_ITEMS;
    S agg{op.identity(), 0};
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++) {
      const int64_t i = base + k;
      if (i < n) agg = seg_combine(op, agg, S{op.elem(i), (uint64_t)(flags[i] & F_PART)});
    }
    int cur = 0;
    s_scan[0][threadIdx.x] = agg;
    __syncthreads();
    for (int off = 1; off < WIN_NT; off <<= 1) {
      S x = s_scan[cur][threadIdx.x];
      if ((int)threadIdx.x >= off) x = seg_combine(op, s_scan[cur][threadIdx.x - off], x);
      s_scan[cur ^ 1][threadIdx.x] = x;
      cur ^= 1;
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const S tile_agg = s_scan[cur][WIN_NT - 1];
      S excl{carry_in ? *carry_in : op.identity(), 0};
      if (tile > 0) {
        t_agg[tile] = tile_agg;
        __threadfence();
        st_volatile_u32(&status[tile], TS_AGG);
        S acc{op.identity(), 0};
        for (int64_t p = tile - 1;; p--) {
          uint32_t st;
          do { st = ld_volatile_u32(&status[p]); } while (st == 0);
          __threadfence();
          if (st == TS_PREFIX) { acc = seg_combine(op, ld_cg(&t_inc[p]), acc); break; }
          const S a = ld_cg(&t_agg[p]);
          acc = seg_combine(op, a, acc);
          if (a.f) break;   // a partition starts in tile p: nothing before it counts
        }
        excl = acc;
      }
      const S inc = seg_combine(op, excl, tile_agg);
      t_inc[tile] = inc;
      __threadfence();
      st_volatile_u32(&status[tile], TS_PREFIX);
      if (tile == ntiles - 1) *carry_out = inc.v;
      s_excl = excl;
    }
    __syncthreads();
    S run = s_excl;
    if (threadIdx.x > 0) run = seg_combine(op, run, s_scan[cur][threadIdx.x - 1]);
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++) {
      const int64_t i = base + k;
      if (i < n) { run = seg_combine(op, run, S{op.elem(i), (uint64_t)(flags[i] & F_PART)}); state[i] = run.v; }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// frames
enum { FR_ROWS_RUNNING = 0, FR_RANGE_RUNNING = 1, FR_GENERAL = 2, FR_RANGE_VALUE = 3 };
struct FrameArgs {
  int32_t type, lower_unb, upper_unb;
  int64_t lower, upper;
};
struct Groups {
  const RankOp::T* rank;
  const int32_t* pend_at;       // partition end, stored at the partition's first row
  const int32_t* peer_end_at;   // peer group end, stored at the peer group's first row
};

__global__ void window_group_ends_kernel(const uint8_t* __restrict__ flags, const RankOp::T* __restrict__ rank, int64_t n, int32_t* __restrict__ pend_at,
                                         int32_t* __restrict__ peer_end_at) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t nf = j == n - 1 ? (F_PART | F_PEER) : flags[j + 1];
    const RankOp::T r = rank[j];
    if (pend_at && (nf & F_PART)) pend_at[max((int64_t)0, j - r.rn + 1)] = (int32_t)j;
    if (peer_end_at && (nf & F_PEER)) peer_end_at[max((int64_t)0, j - r.rn + r.rk)] = (int32_t)j;
  }
}

// The rows a finish or LEAD / LAG launch writes: every row of the chunk, or only [lo, hi) (the rest are context and look-ahead
// rows of a streamed bounded plan, read but never written), into columns of hi - lo rows
struct AllRows {
  int64_t n;
  __device__ __forceinline__ int64_t begin() const { return 0; }
  __device__ __forceinline__ int64_t end() const { return n; }
  __device__ __forceinline__ int64_t out(int64_t i) const { return i; }
};
struct RowRange {
  int64_t lo, hi;
  __device__ __forceinline__ int64_t begin() const { return lo; }
  __device__ __forceinline__ int64_t end() const { return hi; }
  __device__ __forceinline__ int64_t out(int64_t i) const { return i - lo; }
};

// With a carry, rank[i].rn counts from the partition's true start, so ps = i - rn + 1 is clipped to 0 for a partition that began
// in an earlier chunk, and pend_at[0] is then the chunk's last row of it.  Over RowRange rows of a streamed bounded plan neither
// cuts a frame short: the chunk holds P + 1 rows before lo (or every row since the input began, when ps is exact) and F rows
// after hi - 1 (or every row up to the input's end, when pe is exact), so every output row has i + lower >= 1 and
// i + upper <= n - 1.  So s = i + lower >= 1 > ps whenever ps was clipped: such a frame is never from_start and its difference
// of prefixes reads state[s - 1] inside the chunk, where both prefixes include the carry alike.  A frame from UNBOUNDED
// PRECEDING is from_start and reads state[e], which continues the carry as a running frame does.
template <class Op, class R>
__global__ void window_finish_kernel(const Op op, const FrameArgs fr, const Groups g, const typename Op::T* __restrict__ state, const R rows,
                                     const WinOut out) {
  using T = typename Op::T;
  for (int64_t i = rows.begin() + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows.end(); i += (int64_t)gridDim.x * blockDim.x) {
    int64_t s = 0, e = i;
    bool from_start = true, empty = false;
    if (fr.type == FR_RANGE_RUNNING) {
      const RankOp::T r = g.rank[i];
      e = g.peer_end_at[max((int64_t)0, i - r.rn + r.rk)];
    } else if (fr.type == FR_GENERAL) {
      const int64_t ps = max((int64_t)0, i - g.rank[i].rn + 1), pe = g.pend_at[ps];
      s = fr.lower_unb ? ps : max(ps, i + fr.lower);
      e = fr.upper_unb ? pe : min(pe, i + fr.upper);
      from_start = s == ps;
      empty = s > e;
    }
    T v;
    if (empty) v = op.identity();
    else if (from_start) v = state[e];
    else if (Op::SUB) v = op.sub(state[e], state[s - 1]);
    else {
      v = op.identity();
      for (int64_t j = s; j <= e; j++) v = op.combine(v, op.elem(j));
    }
    op.finish(v, fr.type != FR_GENERAL, out, rows.out(i));
  }
}

// map[out(i)] = the source row of row i in the chunk, or -1 outside the partition
template <class R>
__global__ void window_lead_lag_kernel(const RankOp::T* __restrict__ rank, const int32_t* __restrict__ pend_at, const R rows, int64_t off,
                                       int32_t* __restrict__ map) {
  for (int64_t i = rows.begin() + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows.end(); i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ps = max((int64_t)0, i - rank[i].rn + 1), pe = pend_at[ps], src = i + off;
    map[rows.out(i)] = (src >= ps && src <= pe) ? (int32_t)src : -1;
  }
}

// LEAD / LAG default (fixed width) in the rows whose source lies outside the partition
__global__ void window_default_kernel(const int32_t* __restrict__ map, int64_t n, int width, uint4 dflt, void* __restrict__ data, uint32_t* __restrict__ valid) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (map[i] >= 0) continue;
    memcpy(reinterpret_cast<char*>(data) + i * width, &dflt, width);
    atomicOr(&valid[i >> 5], 1u << (i & 31));
  }
}

// ------------------------------------------------------------------------------------------------
// FIRST / LAST / NTH_VALUE (GpuFirst / GpuLast / GpuNthValue: RollingAggregation.nth with a NullPolicy): each row's source row
// in a map, the values then gathered through it

// dir[w] = the valid rows of validity words [0, w): per-word popcounts here (padding bits past row n - 1 masked), then an
// exclusive scan that also writes dir[nwords]
__global__ void window_valid_popc_kernel(const uint32_t* __restrict__ valid, int64_t n, int64_t nwords, int32_t* __restrict__ cnt) {
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
    const int tail = (int)(n - w * 32);
    cnt[w] = __popc(tail >= 32 ? valid[w] : valid[w] & ((1u << tail) - 1));
  }
}

struct ValueFn {
  int32_t last;            // LAST; otherwise FIRST (nth = 1) or NTH_VALUE
  int64_t nth;
  const uint32_t* valid;   // with dir: the column's validity words
  const int32_t* dir;      // IGNORE NULLS over a column with NULLs: the rank directory; null: every row counts
  int64_t n;               // the chunk's rows, also the source row that stands for the carried value
  const int64_t* c0;       // the carried count: the open partition's counted rows before row 0, or null

  // counted rows in [0, x), 0 <= x <= n
  __device__ __forceinline__ int64_t before(int64_t x) const {
    const int64_t w = x >> 5;
    const int b = (int)(x & 31);
    return dir[w] + (b ? __popc(valid[w] & ((1u << b) - 1)) : 0);
  }
  // the row of the counted row of rank t (0-based, t < the chunk's count): the word w with dir[w] <= t < dir[w + 1], galloped for
  // from word `from` in whichever direction holds it and then bisected, so the work grows with the log of the distance; then the
  // (t - dir[w] + 1)-th set bit of the word
  __device__ int64_t select(int64_t t, int64_t from) const {
    const int64_t nw = (n + 31) >> 5;
    int64_t lo, hi;   // dir[lo] <= t < dir[hi]
    if (dir[from] <= t) {
      lo = from;
      for (int64_t d = 1;; d <<= 1) {
        hi = min(from + d, nw);
        if (dir[hi] > t) break;
        lo = hi;
      }
    } else {
      hi = from;
      for (int64_t d = 1;; d <<= 1) {
        lo = max(from - d, (int64_t)0);
        if (dir[lo] <= t) break;
        hi = lo;
      }
    }
    while (hi - lo > 1) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (dir[mid] <= t) lo = mid;
      else hi = mid;
    }
    return lo * 32 + __fns(valid[lo], 0, (int)(t - dir[lo]) + 1);
  }
  // The source row of the frame [s, e] (s <= e unless cont), -1 for NULL, n for the carried value.  cont: the frame starts
  // where the partition does, before row 0 (s = 0); then c0 rows came before it.  e >= 0 there, as a continuing frame always
  // reaches row 0 (running frames; a bounded chunk's output rows have i + upper >= 1).
  __device__ int64_t src(int64_t s, int64_t e, bool cont) const {
    const int64_t c = cont && c0 ? *c0 : 0;
    if (last) {
      if (!dir) return e;
      const int64_t k = before(e + 1);
      if (k > before(s)) return select(k - 1, e >> 5);
      return c > 0 ? n : -1;
    }
    if (c >= nth) return n;
    const int64_t k = nth - c;   // the k-th counted row from s
    if (!dir) return s + k - 1 <= e ? s + k - 1 : -1;
    const int64_t t = before(s) + k - 1;
    return t < before(e + 1) ? select(t, s >> 5) : -1;
  }
};

// map[out(i)] = the source row of row i's frame, found as window_finish_kernel finds [s, e] (RANGE_VALUE: s_at, e_at)
template <class R>
__global__ void window_value_kernel(const ValueFn f, const FrameArgs fr, const Groups g, const int32_t* __restrict__ s_at,
                                    const int32_t* __restrict__ e_at, const R rows, int32_t* __restrict__ map) {
  for (int64_t i = rows.begin() + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows.end(); i += (int64_t)gridDim.x * blockDim.x) {
    const RankOp::T r = g.rank[i];
    const int64_t p = i - r.rn + 1, ps = max((int64_t)0, p);
    int64_t s = ps, e = i;
    bool from_ps = true;
    if (fr.type == FR_RANGE_RUNNING) {
      e = g.peer_end_at[max((int64_t)0, i - r.rn + r.rk)];
    } else if (fr.type == FR_GENERAL) {
      const int64_t pe = g.pend_at[ps];
      s = fr.lower_unb ? ps : max(ps, i + fr.lower);
      e = fr.upper_unb ? pe : min(pe, i + fr.upper);
      from_ps = fr.lower_unb;
    } else if (fr.type == FR_RANGE_VALUE) {
      s = s_at[i];
      e = e_at[i];
      from_ps = false;
    }
    const bool cont = from_ps && p < 0;
    map[rows.out(i)] = (!cont && s > e) ? -1 : (int32_t)f.src(s, e, cont);
  }
}

// the carry at row r (one thread): the count of the open partition's counted rows up to r, and the source row of the value its
// continuing frames resolve to (the frame [partition start, r])
__global__ void window_value_carry_kernel(const ValueFn f, const RankOp::T* __restrict__ rank, int64_t r, int64_t* __restrict__ count,
                                          int32_t* __restrict__ map) {
  const int64_t p = r - rank[r].rn + 1, s = max((int64_t)0, p);
  const bool cont = p < 0;
  *count = (cont && f.c0 ? *f.c0 : 0) + (f.dir ? f.before(r + 1) - f.before(s) : r - s + 1);
  *map = (int32_t)f.src(s, r, cont);
}

// the rows whose source is the carried value (map[i] == mark; the gather left them NULL) take its bytes and validity
__global__ void window_value_patch_kernel(const int32_t* __restrict__ map, int64_t m, int32_t mark, const void* __restrict__ cdata,
                                          const uint32_t* __restrict__ cvalid, int width, void* __restrict__ data, uint32_t* __restrict__ valid) {
  if (!row_valid(cvalid, 0)) return;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    if (map[i] != mark) continue;
    memcpy(reinterpret_cast<char*>(data) + i * width, cdata, width);
    atomicOr(&valid[i >> 5], 1u << (i & 31));
  }
}

// ------------------------------------------------------------------------------------------------
// RANGE frames with value offsets (Spark's RangeBoundOrdering)

// The first ORDER BY column as a key that ascends in the sort order: x, or -x for DESC, exact in 128 bits, so that the bound
// values key(i) + lower and key(i) + upper never wrap (|x| < 10^38 for decimals, offsets are int64).  A NULL sorts before every
// value (nulls first) or after it.  col.data == null: no value offsets, every bounded side is a peer-group edge.
struct RangeKey {
  ColView col;
  int32_t desc, nulls_first;
  __device__ __forceinline__ i128 at(int64_t j) const {
    const i128 x = col.width == 16 ? reinterpret_cast<const i128*>(col.data)[j] : (i128)load_int(col, j);
    return desc ? -x : x;
  }
  // the first row j of [lo, hi] whose key is >= b (strict: > b), or hi + 1; the keys of [lo, hi] ascend
  __device__ int64_t first_past(int64_t lo, int64_t hi, i128 b, bool strict) const {
    int64_t a = lo, z = hi + 1;
    while (a < z) {
      const int64_t mid = a + ((z - a) >> 1);
      bool past;
      if (!row_valid(col.valid, mid)) past = !nulls_first;
      else {
        const i128 k = at(mid);
        past = strict ? k > b : k >= b;
      }
      if (past) z = mid;
      else a = mid + 1;
    }
    return a;
  }
};
struct RangeBounds {
  int64_t lower, upper;   // value offsets; 0 = the peer-group edge
  int32_t lower_unb, upper_unb;
};

// s[i], e[i]: row i's frame, partition rows only (s > e: empty).  A NULL ORDER BY value's bounds are NULL, so its bounded sides
// are the edges of its (NULL) peer group; a non-NULL value's bounded frame never reaches a NULL row.
__global__ void window_range_bounds_kernel(const RangeKey key, const RangeBounds b, const Groups g, int64_t n, int32_t* __restrict__ s_at,
                                           int32_t* __restrict__ e_at) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const RankOp::T r = g.rank[i];
    const int64_t ps = max((int64_t)0, i - r.rn + 1), pe = g.pend_at[ps];
    const int64_t qs = max((int64_t)0, i - r.rn + r.rk), qe = g.peer_end_at[qs];
    const bool by_peer = key.col.data == nullptr || !row_valid(key.col.valid, i);
    const i128 v = by_peer ? (i128)0 : key.at(i);
    int64_t s, e;
    if (b.lower_unb) s = ps;
    else if (b.lower == 0 || by_peer) s = qs;
    else s = key.first_past(ps, pe, v + (i128)b.lower, false);
    if (b.upper_unb) e = pe;
    else if (b.upper == 0 || by_peer) e = qe;
    else e = key.first_past(ps, pe, v + (i128)b.upper, true) - 1;
    s_at[i] = (int32_t)s;
    e_at[i] = (int32_t)e;
  }
}

// the range-query structure of a non-SUB op over a chunk (unsegmented: a frame never leaves its partition)
template <typename T>
struct RangeTable {
  const T* pre;      // pre[i]: rows [tile start, i]
  const T* suf;      // suf[i]: rows [i, tile end]
  const T* levels;   // levels[k * ntiles + t]: tiles [t, t + 2^k)
  int64_t ntiles;
  int32_t nlevels;
};

template <class Op>
__global__ void __launch_bounds__(WIN_NT) window_range_tiles_kernel(const Op op, int64_t n, typename Op::T* __restrict__ pre, typename Op::T* __restrict__ suf,
                                                                    typename Op::T* __restrict__ agg) {
  using T = typename Op::T;
  __shared__ T s_scan[2][WIN_NT];
  const int64_t ntiles = (n + WIN_TILE - 1) / WIN_TILE;
  const int tx = threadIdx.x;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * WIN_TILE + (int64_t)tx * WIN_ITEMS;
    T a = op.identity();
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++)
      if (base + k < n) a = op.combine(a, op.elem(base + k));
    // prefix: inclusive scan of the thread aggregates from the left
    int cur = 0;
    s_scan[0][tx] = a;
    __syncthreads();
    for (int off = 1; off < WIN_NT; off <<= 1) {
      T y = s_scan[cur][tx];
      if (tx >= off) y = op.combine(s_scan[cur][tx - off], y);
      s_scan[cur ^ 1][tx] = y;
      cur ^= 1;
      __syncthreads();
    }
    T run = tx > 0 ? s_scan[cur][tx - 1] : op.identity();
    if (tx == WIN_NT - 1) agg[tile] = s_scan[cur][tx];
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++)
      if (base + k < n) { run = op.combine(run, op.elem(base + k)); pre[base + k] = run; }
    __syncthreads();
    // suffix: the same from the right
    cur = 0;
    s_scan[0][tx] = a;
    __syncthreads();
    for (int off = 1; off < WIN_NT; off <<= 1) {
      T y = s_scan[cur][tx];
      if (tx + off < WIN_NT) y = op.combine(y, s_scan[cur][tx + off]);
      s_scan[cur ^ 1][tx] = y;
      cur ^= 1;
      __syncthreads();
    }
    run = tx < WIN_NT - 1 ? s_scan[cur][tx + 1] : op.identity();
#pragma unroll
    for (int k = WIN_ITEMS - 1; k >= 0; k--)
      if (base + k < n) { run = op.combine(op.elem(base + k), run); suf[base + k] = run; }
    __syncthreads();
  }
}

// level k of the sparse table from level k - 1 (half = 2^(k-1)); entries that would pass the last tile are never read
template <class Op>
__global__ void window_range_table_kernel(const Op op, int64_t ntiles, int64_t half, const typename Op::T* __restrict__ prev,
                                          typename Op::T* __restrict__ next) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < ntiles; t += (int64_t)gridDim.x * blockDim.x)
    next[t] = t + half < ntiles ? op.combine(prev[t], prev[t + half]) : prev[t];
}

// the op over rows [s, e] (s <= e) through the structure: at most WIN_TILE elements, or two reads and one per level
template <class Op>
__device__ __forceinline__ typename Op::T range_query(const Op& op, const RangeTable<typename Op::T>& rt, int64_t s, int64_t e) {
  using T = typename Op::T;
  const int64_t ts = s / WIN_TILE, te = e / WIN_TILE;
  if (ts == te) {
    T v = op.identity();
    for (int64_t j = s; j <= e; j++) v = op.combine(v, op.elem(j));
    return v;
  }
  // the whole tiles [ts + 1, te) in blocks of decreasing powers of two, each level at most once
  T v = rt.suf[s];
  int64_t a = ts + 1;
  for (int k = rt.nlevels - 1; k >= 0; k--)
    if (a + ((int64_t)1 << k) <= te) {
      v = op.combine(v, rt.levels[(int64_t)k * rt.ntiles + a]);
      a += (int64_t)1 << k;
    }
  return op.combine(v, rt.pre[e]);
}

// Every row of a chunk that starts at a partition start (a RANGE_VALUE plan holds whole partitions), from s[i] and e[i]
template <class Op>
__global__ void window_range_finish_kernel(const Op op, const Groups g, const int32_t* __restrict__ s_at, const int32_t* __restrict__ e_at,
                                           const typename Op::T* __restrict__ state, const RangeTable<typename Op::T> rt, int64_t n, const WinOut out) {
  using T = typename Op::T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ps = max((int64_t)0, i - g.rank[i].rn + 1), s = s_at[i], e = e_at[i];
    T v;
    if (s > e) v = op.identity();
    else if (s == ps) v = state[e];
    else if (Op::SUB) v = op.sub(state[e], state[s - 1]);
    else v = range_query(op, rt, s, e);
    op.finish(v, false, out, i);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
static bool is_ranking(int k) { return k == B2_WIN_ROW_NUMBER || k == B2_WIN_RANK || k == B2_WIN_DENSE_RANK; }
static bool is_offset_fn(int k) { return k == B2_WIN_LEAD || k == B2_WIN_LAG; }
static bool is_value_fn(int k) { return k == B2_WIN_FIRST || k == B2_WIN_LAST || k == B2_WIN_NTH_VALUE; }
static bool needs_column(int k) { return !is_ranking(k) && k != B2_WIN_COUNT_ALL; }
// a RANGE_VALUE bound that is a value offset (not CURRENT ROW, not UNBOUNDED)
static bool value_offset(int64_t b) { return b != 0 && b != B2_UNBOUNDED_PRECEDING && b != B2_UNBOUNDED_FOLLOWING; }

// checks what the specs say about themselves and classifies the frames; column types are checked by bind()
WindowPlan make_window_plan(const int32_t* part_cols, int nparts, const b2_order_by_arg* order, int norder, const b2_window_spec* specs, int nspecs) {
  B2_CHECK(nparts >= 0 && norder >= 0 && nspecs >= 1, "window: bad number of partition keys, order keys or functions");
  B2_CHECK(nparts <= SORT_MAX_KEYS && norder <= SORT_MAX_KEYS, "window: too many keys");
  WindowPlan p;
  p.part.assign(part_cols, part_cols + nparts);
  p.order.assign(order, order + norder);
  p.mode = 1;
  // the row extents of the streamed bounded class: offsets clamped as frame_args clamps them, so P + F cannot overflow
  const int64_t lim = (int64_t)1 << 40;
  auto clamp = [&](int64_t v) { return std::max(-lim, std::min(lim, v)); };
  bool streamable = true;
  for (int k = 0; k < nspecs; k++) {
    WinFn f;
    f.s = specs[k];
    const int kind = f.s.kind;
    if (f.s.ignore_nulls && !is_value_fn(kind)) {
      if (is_offset_fn(kind)) throw Error(B2_ERR_UNSUPPORTED, "window: LEAD / LAG IGNORE NULLS");
      throw Error(B2_ERR_INVALID, "window: IGNORE NULLS on a function other than FIRST / LAST / NTH_VALUE");
    }
    if (is_ranking(kind) || is_offset_fn(kind)) {
      B2_CHECK(norder > 0, "window: ranking functions and LEAD / LAG need ORDER BY");
      f.frame = FR_ROWS_RUNNING;
      if (is_offset_fn(kind)) {
        B2_CHECK(f.s.offset >= 0, "window: LEAD / LAG offset must be >= 0");
        f.frame = FR_GENERAL;
      }
    } else if (kind == B2_WIN_SUM || kind == B2_WIN_COUNT || kind == B2_WIN_COUNT_ALL || kind == B2_WIN_MIN || kind == B2_WIN_MAX || is_value_fn(kind)) {
      B2_CHECK(kind != B2_WIN_NTH_VALUE || f.s.offset >= 1, "window: NTH_VALUE needs n >= 1");
      const bool lu = f.s.lower == B2_UNBOUNDED_PRECEDING, uu = f.s.upper == B2_UNBOUNDED_FOLLOWING;
      B2_CHECK(f.s.frame == B2_FRAME_ROWS || f.s.frame == B2_FRAME_RANGE || f.s.frame == B2_FRAME_RANGE_VALUE, "window: unknown frame type");
      B2_CHECK(f.s.lower != B2_UNBOUNDED_FOLLOWING && f.s.upper != B2_UNBOUNDED_PRECEDING, "window: frame bounds in the wrong direction");
      B2_CHECK(lu || uu || f.s.lower <= f.s.upper, "window: frame lower bound above the upper bound");
      if (f.s.frame == B2_FRAME_RANGE && !(lu && (uu || f.s.upper == 0)))
        throw Error(B2_ERR_UNSUPPORTED, "window: RANGE frames with value offsets");
      if (f.s.frame == B2_FRAME_RANGE_VALUE) {
        B2_CHECK(norder > 0 || (lu && uu), "window: a RANGE frame bounded by value needs ORDER BY");
        B2_CHECK(norder == 1 || !(value_offset(f.s.lower) || value_offset(f.s.upper)), "window: RANGE value offsets need exactly one ORDER BY column");
      }
      // RANGE_VALUE (UNBOUNDED, 0) and (UNBOUNDED, UNBOUNDED) are RANGE's running and whole-partition frames
      if (lu && f.s.upper == 0) f.frame = f.s.frame == B2_FRAME_ROWS ? FR_ROWS_RUNNING : FR_RANGE_RUNNING;
      else if (f.s.frame == B2_FRAME_RANGE_VALUE && !(lu && uu)) f.frame = FR_RANGE_VALUE;
      else f.frame = FR_GENERAL;
    } else {
      throw Error(B2_ERR_INVALID, "window: unknown function kind " + std::to_string(kind));
    }
    const int m = (f.frame == FR_GENERAL || f.frame == FR_RANGE_VALUE) ? 3 : f.frame == FR_RANGE_RUNNING ? 2 : 1;
    p.mode = std::max(p.mode, m);
    if (kind == B2_WIN_LAG) p.pre = std::max(p.pre, (int64_t)f.s.offset);
    else if (kind == B2_WIN_LEAD) p.post = std::max(p.post, (int64_t)f.s.offset);
    else if (!is_ranking(kind)) {
      if (f.s.frame != B2_FRAME_ROWS || f.s.upper == B2_UNBOUNDED_FOLLOWING) {
        streamable = false;
      } else {
        // UNBOUNDED PRECEDING -> u reads the scan state at row i + u; [l, u] reads the rows between i + l and i + u
        const int64_t u = clamp(f.s.upper), l = f.s.lower == B2_UNBOUNDED_PRECEDING ? u : clamp(f.s.lower);
        p.pre = std::max(p.pre, std::max(-l, -u));
        p.post = std::max(p.post, std::max(l, u));
      }
    }
    p.fns.push_back(f);
  }
  p.bounded = streamable && p.pre + p.post > 0;
  return p;
}

// the columns the plan reads (partition keys, order keys, function inputs; each once) and the plan over a table of just those
std::vector<int> window_read_columns(const WindowPlan& p, WindowPlan* over_read) {
  std::vector<int> cols;
  auto at = [&](int c) -> int32_t {
    for (size_t k = 0; k < cols.size(); k++)
      if (cols[k] == c) return (int32_t)k;
    cols.push_back(c);
    return (int32_t)cols.size() - 1;
  };
  *over_read = p;
  for (int32_t& c : over_read->part) c = at(c);
  for (auto& o : over_read->order) o.column = at(o.column);
  for (WinFn& f : over_read->fns)
    if (needs_column(f.s.kind)) f.s.column = at(f.s.column);
  return cols;
}

// checks the columns of the first batch against the plan
void bind_window(WindowPlan& p, const Table* t) {
  const int nc = (int)t->cols.size();
  for (int32_t c : p.part) B2_CHECK(c >= 0 && c < nc, "window: partition key column out of range");
  for (auto& o : p.order) B2_CHECK(o.column >= 0 && o.column < nc, "window: order key column out of range");
  for (WinFn& f : p.fns) {
    const int kind = f.s.kind;
    if (f.frame == FR_RANGE_VALUE && (value_offset(f.s.lower) || value_offset(f.s.upper))) {
      const int ot = t->cols[p.order[0].column]->dtype;
      if (is_float(ot)) throw Error(B2_ERR_UNSUPPORTED, "window: RANGE value offsets over a FLOAT ORDER BY column");
      B2_CHECK(ot == B2_INT8 || ot == B2_INT16 || ot == B2_INT32 || ot == B2_INT64 || ot == B2_DATE32 || ot == B2_TIMESTAMP_US || is_decimal(ot),
               "window: RANGE value offsets need an integer, DATE32, TIMESTAMP_US or decimal ORDER BY column");
    }
    if (!needs_column(kind)) continue;
    B2_CHECK(f.s.column >= 0 && f.s.column < nc, "window: function column out of range");
    const int dt = t->cols[f.s.column]->dtype;
    f.in_dtype = dt;
    if (is_offset_fn(kind)) {
      if (dt == B2_STRING && !f.s.default_is_null) throw Error(B2_ERR_UNSUPPORTED, "window: LEAD / LAG default on a STRING column");
    } else if (kind == B2_WIN_SUM) {
      if (is_decimal(dt)) {
        B2_CHECK(f.s.out_dtype == B2_DECIMAL128 || (f.s.out_dtype == B2_DECIMAL64 && f.s.out_precision <= 18), "window: decimal SUM needs a decimal result type");
        B2_CHECK(f.s.out_precision >= 1 && f.s.out_precision <= 38, "window: decimal SUM needs out_precision in 1..38");
      } else if (!(dt == B2_INT8 || dt == B2_INT16 || dt == B2_INT32 || dt == B2_INT64 || is_float(dt))) {
        throw Error(B2_ERR_UNSUPPORTED, "window: SUM over dtype " + std::to_string(dt));
      }
    } else if (kind == B2_WIN_MIN || kind == B2_WIN_MAX) {
      if (dt == B2_STRING || dt == B2_DECIMAL128) throw Error(B2_ERR_UNSUPPORTED, "window: MIN / MAX over STRING or DECIMAL128");
    }
  }
}

template <class Op>
static DevBuf run_scan(const Op& op, const uint8_t* flags, int64_t n, const DevBuf* carry_in, DevBuf& carry_out) {
  using T = typename Op::T;
  DevBuf state((size_t)n * sizeof(T));
  carry_out = DevBuf(sizeof(T));
  const int64_t ntiles = (n + WIN_TILE - 1) / WIN_TILE;
  DevBuf work(8 + (size_t)ntiles * 4);
  CUDA_CHECK(cudaMemsetAsync(work.p, 0, work.bytes, stream()));
  DevBuf agg((size_t)ntiles * sizeof(Seg<T>)), inc((size_t)ntiles * sizeof(Seg<T>));
  launch("window_scan_kernel", window_scan_kernel<Op>, grid_for(ntiles, 1, 8), WIN_NT, 0, stream(), op, flags, n, state.as<T>(),
         carry_in && carry_in->p ? carry_in->as<T>() : (const T*)nullptr, carry_out.as<T>(), work.as<unsigned long long>(),
         reinterpret_cast<uint32_t*>(work.as<char>() + 8), agg.as<Seg<T>>(), inc.as<Seg<T>>());
  return state;
}

// the output rows of a chunk and the row the carry is taken at (rows = null: every row, carry at the last)
struct ChunkRows { int64_t lo, hi, carry_row; };

template <class Op>
static void run_finish(const Op& op, const FrameArgs& fr, const Groups& g, const DevBuf& state, int64_t n, const WinOut& o, const ChunkRows* rows) {
  using T = typename Op::T;
  if (!rows) launch("window_finish_kernel", window_finish_kernel<Op, AllRows>, grid_for(n, 256), 256, 0, stream(), op, fr, g, state.as<T>(), AllRows{n}, o);
  else launch("window_finish_kernel", window_finish_kernel<Op, RowRange>, grid_for(rows->hi - rows->lo, 256), 256, 0, stream(), op, fr, g, state.as<T>(),
              RowRange{rows->lo, rows->hi}, o);
}

// a RANGE_VALUE function over every row of a chunk, from its frames se = [s[0..n), e[0..n)]
template <class Op>
static void run_range_finish(const Op& op, const Groups& g, const DevBuf& se, const DevBuf& state, int64_t n, const WinOut& o) {
  using T = typename Op::T;
  RangeTable<T> rt{nullptr, nullptr, nullptr, 0, 0};
  DevBuf pre, suf, levels;
  if constexpr (!Op::SUB) {
    // 2 n + ~n / 512 states: 32 B per row for a 16-byte state
    const int64_t ntiles = (n + WIN_TILE - 1) / WIN_TILE;
    int nlev = 1;
    while (((int64_t)1 << nlev) <= ntiles) nlev++;
    pre = DevBuf((size_t)n * sizeof(T));
    suf = DevBuf((size_t)n * sizeof(T));
    levels = DevBuf((size_t)nlev * ntiles * sizeof(T));
    T* lv = levels.as<T>();
    launch("window_range_tiles_kernel", window_range_tiles_kernel<Op>, grid_for(ntiles, 1, 8), WIN_NT, 0, stream(), op, n, pre.as<T>(), suf.as<T>(), lv);
    for (int k = 1; k < nlev; k++)
      launch("window_range_table_kernel", window_range_table_kernel<Op>, grid_for(ntiles, 256), 256, 0, stream(), op, ntiles, (int64_t)1 << (k - 1),
             (const T*)(lv + (int64_t)(k - 1) * ntiles), lv + (int64_t)k * ntiles);
    rt = RangeTable<T>{pre.as<T>(), suf.as<T>(), lv, ntiles, nlev};
  }
  const int32_t* s = se.as<int32_t>();
  launch("window_range_finish_kernel", window_range_finish_kernel<Op>, grid_for(n, 256), 256, 0, stream(), op, g, s, s + n, state.as<T>(), rt, n, o);
}

static SortPlan empty_plan() { SortPlan p; memset(&p, 0, sizeof(p)); return p; }

// boundary flags of `t` (row 0 against `last` when given)
static DevBuf window_flags(const WindowPlan& p, const Table* t, const Table* last) {
  const int64_t n = t->rows;
  std::vector<b2_order_by_arg> pk;
  for (int32_t c : p.part) pk.push_back(b2_order_by_arg{c, 1, 1});
  SortPlan part = empty_plan(), order = empty_plan(), cpart = empty_plan(), corder = empty_plan();
  if (last) {
    if (!pk.empty()) { auto v = shared_sort_plans({t, last}, pk.data(), (int)pk.size()); part = v[0]; cpart = v[1]; }
    if (!p.order.empty()) { auto v = shared_sort_plans({t, last}, p.order.data(), (int)p.order.size()); order = v[0]; corder = v[1]; }
  } else {
    if (!pk.empty()) part = make_sort_plan(t, pk.data(), (int)pk.size());
    if (!p.order.empty()) order = make_sort_plan(t, p.order.data(), (int)p.order.size());
  }
  DevBuf flags((size_t)std::max<int64_t>(n, 1));
  if (n) launch("window_bounds_kernel", window_bounds_kernel, grid_for(n, 256), 256, 0, stream(), part, order, cpart, corder, last ? 1 : 0, n, flags.as<uint8_t>());
  return flags;
}

// the last row of `t` whose flags have a bit of mask, or -1 (one device-to-host copy)
int64_t window_last_start(const WindowPlan& p, const Table* t, const Table* last, uint8_t mask) {
  DevBuf flags = window_flags(p, t, last);
  DevBuf out(8);
  CUDA_CHECK(cudaMemsetAsync(out.p, 0xff, 8, stream()));
  launch("window_last_start_kernel", window_last_start_kernel, grid_for(t->rows, 256), 256, 0, stream(), flags.as<uint8_t>(), t->rows, mask,
         out.as<unsigned long long>());
  int64_t h = -1;
  d2h(&h, out.p, 1);
  sync();
  return h;
}

static FrameArgs frame_args(const WinFn& f) {
  FrameArgs fr;
  fr.type = f.frame;
  fr.lower_unb = f.s.lower == B2_UNBOUNDED_PRECEDING;
  fr.upper_unb = f.s.upper == B2_UNBOUNDED_FOLLOWING;
  const int64_t lim = (int64_t)1 << 40;   // beyond any batch; keeps i + bound from overflowing
  fr.lower = std::max(-lim, std::min(lim, f.s.lower));
  fr.upper = std::max(-lim, std::min(lim, f.s.upper));
  return fr;
}

// the state at row r of a scan (r >= 0) as the carry of that function, copied on the device
template <typename T>
static void carry_at(const DevBuf& state, int64_t r, DevBuf& carry) {
  CUDA_CHECK(cudaMemcpyAsync(carry.p, state.as<char>() + (size_t)r * sizeof(T), sizeof(T), cudaMemcpyDeviceToDevice, stream()));
}

// Column c of t gathered through map (m rows, out of range = NULL) as a value function's result; the rows whose source is t->rows
// take cv, the one-row carried value
static Column* gather_values(const Table* t, int c, const int32_t* map, int64_t m, const Column* cv) {
  using TablePtr = std::unique_ptr<Table, void (*)(Table*)>;
  const std::vector<int> only{c};
  Column* oc;
  if (cv && t->cols[c]->dtype == B2_STRING) {
    // a STRING carried value is gathered from the column with it appended as row t->rows (a copy of the column's offsets and
    // chars); a fixed-width column is never copied, its carried rows are patched below
    Column *a = t->cols[c], *b = const_cast<Column*>(cv);
    col_incref(a);
    col_incref(b);
    TablePtr ta(new_table({a}), table_release), tb(new_table({b}), table_release);
    TablePtr both(concat_tables({ta.get(), tb.get()}), table_release);
    TablePtr got(gather_table(both.get(), map, m, true, nullptr), table_release);
    oc = got->cols[0];
    col_incref(oc);
  } else {
    TablePtr got(gather_table(t, map, m, true, &only), table_release);
    oc = got->cols[0];
    col_incref(oc);
    if (cv && m)
      launch("window_value_patch_kernel", window_value_patch_kernel, grid_for(m, 256), 256, 0, stream(), map, m, (int32_t)t->rows, (const void*)cv->data.p,
             cv->validity(), dtype_width(oc->dtype), oc->data.p, oc->valid.as<uint32_t>());
  }
  finalize_nulls(oc);
  return oc;
}

// The functions over one chunk of rows sorted by (partition, order), one column per function.  With `rows`, only the rows
// [lo, hi) are written (columns of hi - lo rows) and the carry is taken at rows->carry_row (-1: the carry passed in stays);
// otherwise every row, and the carry at the last row.  The carry is replaced only on success.
static std::vector<Column*> window_functions(WindowPlan& p, const Table* t, WindowCarry* carry, const ChunkRows* rows) {
  const int64_t n = t->rows;
  if (n > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "window over more than 2^31-1 rows");
  const int64_t lo = rows ? rows->lo : 0, hi = rows ? rows->hi : n, m = hi - lo;
  const int64_t carry_row = rows ? rows->carry_row : n - 1;
  const size_t nf = p.fns.size();
  const Table* last = carry ? carry->last : nullptr;
  const bool has_state = carry && !carry->state.empty();
  DevBuf flags = window_flags(p, t, last);
  std::vector<DevBuf> next_state(nf + 1);
  const uint8_t* fl = flags.as<uint8_t>();

  RankOp rop{fl};
  DevBuf rank = n ? run_scan(rop, fl, n, has_state ? &carry->state[0] : nullptr, next_state[0]) : DevBuf();
  if (rows && carry_row >= 0) carry_at<RankOp::T>(rank, carry_row, next_state[0]);
  bool need_pend = false, need_peer = false;
  for (const WinFn& f : p.fns) {
    need_pend = need_pend || f.frame == FR_GENERAL || f.frame == FR_RANGE_VALUE;
    need_peer = need_peer || f.frame == FR_RANGE_RUNNING || f.frame == FR_RANGE_VALUE;
  }
  DevBuf pend, peer;
  if (n && (need_pend || need_peer)) {
    if (need_pend) pend = DevBuf((size_t)n * 4);
    if (need_peer) peer = DevBuf((size_t)n * 4);
    launch("window_group_ends_kernel", window_group_ends_kernel, grid_for(n, 256), 256, 0, stream(), fl, rank.as<RankOp::T>(), n, pend.as<int32_t>(),
           peer.as<int32_t>());
  }
  const Groups g{rank.as<RankOp::T>(), pend.as<int32_t>(), peer.as<int32_t>()};

  // the frames of each distinct RANGE_VALUE (lower, upper), computed once and shared by the functions that use it
  std::vector<std::pair<std::pair<int64_t, int64_t>, DevBuf>> range_frames;
  auto frames_of = [&](const WinFn& f) -> const DevBuf& {
    const std::pair<int64_t, int64_t> key{f.s.lower, f.s.upper};
    for (auto& rf : range_frames)
      if (rf.first == key) return rf.second;
    B2_CHECK(!rows, "window: RANGE frames with value offsets do not stream");
    RangeKey rk{ColView{}, 0, 0};
    if (value_offset(f.s.lower) || value_offset(f.s.upper)) {
      rk.col = view_of(t->cols[p.order[0].column]);
      rk.desc = p.order[0].ascending ? 0 : 1;
      rk.nulls_first = p.order[0].nulls_first ? 1 : 0;
    }
    const RangeBounds b{f.s.lower, f.s.upper, f.s.lower == B2_UNBOUNDED_PRECEDING, f.s.upper == B2_UNBOUNDED_FOLLOWING};
    DevBuf se((size_t)n * 8);
    launch("window_range_bounds_kernel", window_range_bounds_kernel, grid_for(n, 256), 256, 0, stream(), rk, b, g, n, se.as<int32_t>(), se.as<int32_t>() + n);
    range_frames.emplace_back(key, std::move(se));
    return range_frames.back().second;
  };

  // the rank directory of each distinct column that an IGNORE NULLS function reads and that has NULLs, shared likewise
  std::vector<std::pair<int, DevBuf>> dirs;
  auto dir_of = [&](int c) -> const int32_t* {
    for (auto& d : dirs)
      if (d.first == c) return d.second.as<int32_t>();
    const int64_t nw = (n + 31) / 32;
    DevBuf d((size_t)(nw + 1) * 4);
    launch("window_valid_popc_kernel", window_valid_popc_kernel, grid_for(nw, 256), 256, 0, stream(), t->cols[c]->validity(), n, nw, d.as<int32_t>());
    exclusive_scan<int32_t, int32_t>(d.as<int32_t>(), d.as<int32_t>(), nw, true);
    dirs.emplace_back(c, std::move(d));
    return dirs.back().second.as<int32_t>();
  };

  ColsGuard outs, next_value;
  next_value.v.assign(nf + 1, nullptr);
  for (size_t k = 0; k < nf; k++) {
    const WinFn& f = p.fns[k];
    const int kind = f.s.kind;
    const DevBuf* cin = has_state && carry->state[k + 1].p ? &carry->state[k + 1] : nullptr;
    const Column* in = needs_column(kind) ? t->cols[f.s.column] : nullptr;
    if (is_value_fn(kind)) {
      const Column* cv = cin && k + 1 < carry->value.size() ? carry->value[k + 1] : nullptr;
      const ValueFn vf{kind == B2_WIN_LAST ? 1 : 0, kind == B2_WIN_NTH_VALUE ? (int64_t)f.s.offset : 1, in->validity(),
                       n && f.s.ignore_nulls && in->nullable() ? dir_of(f.s.column) : nullptr, n, cin ? cin->as<int64_t>() : nullptr};
      const int32_t* s_at = nullptr;
      if (f.frame == FR_RANGE_VALUE && n) s_at = frames_of(f).as<int32_t>();
      const FrameArgs fr = frame_args(f);
      DevBuf map((size_t)std::max<int64_t>(m, 1) * 4);
      if (m && !rows)
        launch("window_value_kernel", window_value_kernel<AllRows>, grid_for(n, 256), 256, 0, stream(), vf, fr, g, s_at, s_at ? s_at + n : nullptr,
               AllRows{n}, map.as<int32_t>());
      else if (m)
        launch("window_value_kernel", window_value_kernel<RowRange>, grid_for(m, 256), 256, 0, stream(), vf, fr, g, s_at, s_at ? s_at + n : nullptr,
               RowRange{lo, hi}, map.as<int32_t>());
      outs.v.push_back(gather_values(t, f.s.column, map.as<int32_t>(), m, cv));
      if (carry && n && carry_row >= 0) {
        next_state[k + 1] = DevBuf(8);
        DevBuf one(4);
        launch("window_value_carry_kernel", window_value_carry_kernel, 1, 1, 0, stream(), vf, rank.as<RankOp::T>(), carry_row,
               next_state[k + 1].as<int64_t>(), one.as<int32_t>());
        next_value.v[k + 1] = gather_values(t, f.s.column, one.as<int32_t>(), 1, cv);
      }
      continue;
    }
    if (is_offset_fn(kind)) {
      DevBuf map((size_t)std::max<int64_t>(m, 1) * 4);
      const int64_t off = kind == B2_WIN_LEAD ? (int64_t)f.s.offset : -(int64_t)f.s.offset;
      if (m && !rows)
        launch("window_lead_lag_kernel", window_lead_lag_kernel<AllRows>, grid_for(n, 256), 256, 0, stream(), rank.as<RankOp::T>(), pend.as<int32_t>(),
               AllRows{n}, off, map.as<int32_t>());
      else if (m)
        launch("window_lead_lag_kernel", window_lead_lag_kernel<RowRange>, grid_for(m, 256), 256, 0, stream(), rank.as<RankOp::T>(), pend.as<int32_t>(),
               RowRange{lo, hi}, off, map.as<int32_t>());
      std::vector<int> only{f.s.column};
      std::unique_ptr<Table, void (*)(Table*)> got(gather_table(t, map.as<int32_t>(), m, true, &only), table_release);
      Column* c = got->cols[0];
      col_incref(c);
      outs.v.push_back(c);
      if (!f.s.default_is_null && m) {
        uint4 d;
        memcpy(&d, f.s.default_value, 16);
        launch("window_default_kernel", window_default_kernel, grid_for(m, 256), 256, 0, stream(), map.as<int32_t>(), m, dtype_width(c->dtype), d, c->data.p,
               c->valid.as<uint32_t>());
      }
      finalize_nulls(c);
      continue;
    }
    int odt = B2_INT64, oscale = 0;
    if (is_ranking(kind)) odt = B2_INT32;
    else if (kind == B2_WIN_SUM) {
      if (is_decimal(f.in_dtype)) { odt = f.s.out_dtype; oscale = in->scale; }
      else if (is_float(f.in_dtype)) odt = B2_FLOAT64;
    } else if (kind == B2_WIN_MIN || kind == B2_WIN_MAX) { odt = in->dtype; oscale = in->scale; }
    Column* oc = new_column(odt, oscale, m, true);
    outs.v.push_back(oc);
    if (m == 0) { finalize_nulls(oc); continue; }
    CUDA_CHECK(cudaMemsetAsync(oc->valid.p, 0, oc->valid.bytes, stream()));
    const WinOut o{oc->data.p, oc->valid.as<uint32_t>(), odt, f.s.out_precision, kind == B2_WIN_ROW_NUMBER ? 0 : kind == B2_WIN_RANK ? 1 : 2};
    const FrameArgs fr = frame_args(f);
    auto scan_finish = [&](const auto& op) {
      using T = typename std::decay_t<decltype(op)>::T;
      DevBuf st = run_scan(op, fl, n, cin, next_state[k + 1]);
      if (rows && carry_row >= 0) carry_at<T>(st, carry_row, next_state[k + 1]);
      if (f.frame == FR_RANGE_VALUE) run_range_finish(op, g, frames_of(f), st, n, o);
      else run_finish(op, fr, g, st, n, o, rows);
    };
    if (is_ranking(kind)) run_finish(rop, fr, g, rank, n, o, rows);
    else if (kind == B2_WIN_COUNT || kind == B2_WIN_COUNT_ALL) scan_finish(CountOp{in ? view_of(in) : ColView{}, kind == B2_WIN_COUNT_ALL});
    else if (kind == B2_WIN_SUM && is_decimal(f.in_dtype)) scan_finish(SumDecOp{view_of(in)});
    else if (kind == B2_WIN_SUM && is_float(f.in_dtype)) scan_finish(SumFloatOp{view_of(in)});
    else if (kind == B2_WIN_SUM) scan_finish(SumIntOp{view_of(in)});
    else scan_finish(MinMaxOp{view_of(in), kind == B2_WIN_MAX});
    finalize_nulls(oc);
  }
  if (carry && n && carry_row >= 0) {   // replaced only now, so that a failed attempt leaves the carry as it was
    Table* nl = slice_table(t, carry_row, carry_row + 1);
    if (carry->last) table_release(carry->last);
    carry->last = nl;
    carry->state = std::move(next_state);
    for (Column* c : carry->value) if (c) col_release(c);
    carry->value = next_value.release();
  }
  return outs.release();
}

// One chunk of rows sorted by (partition, order): the input columns, then one column per function.  With a carry, row 0 continues
// the partition the previous chunk ended with (when its keys say so) and the carry is replaced by this chunk's on success.
Table* window_chunk(WindowPlan& p, const Table* t, WindowCarry* carry) {
  std::vector<Column*> fns = window_functions(p, t, carry, nullptr);
  ColsGuard outs;
  for (Column* c : t->cols) { col_incref(c); outs.v.push_back(c); }
  outs.v.insert(outs.v.end(), fns.begin(), fns.end());
  return new_table(outs.release());
}

Table* window_chunk_rows(WindowPlan& p, const Table* t, WindowCarry* carry, int64_t lo, int64_t hi, int64_t carry_row) {
  B2_CHECK(lo >= 0 && lo <= hi && hi <= t->rows && carry_row >= -1 && carry_row < t->rows, "window: chunk rows out of range");
  const ChunkRows rows{lo, hi, carry_row};
  return new_table(window_functions(p, t, carry, &rows));
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_window(b2_handle table, const int32_t* part_cols, int32_t nparts, const b2_order_by_arg* order, int32_t norder, const b2_window_spec* specs,
              int32_t nspecs, b2_handle* out_table) {
  B2_TRY
  Table* t = table_from(table);
  WindowPlan p = make_window_plan(part_cols, nparts, order, norder, specs, nspecs);
  bind_window(p, t);
  *out_table = to_handle(window_chunk(p, t, nullptr));
  B2_CATCH
}

}  // extern "C"
