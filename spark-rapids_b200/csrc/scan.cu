// scan.cu — a1 + a2: project and filter as single fused kernels over the VM (vm.cuh).
//
//  project: GpuProjectExec / GpuTieredProject.project (basicPhysicalOperators.scala:116-140,
//           1052-1076) — all bound expressions of the exec evaluated by one launch.
//  filter : GpuFilter.apply / doFilter / computeCheckedFilterMask (:1148-1224).  The reference
//           makes a mask column, reduces it (all()), then runs Table.filter which re-reads the
//           mask for every column.  Here predicate evaluation, the ordered output-offset scan
//           (warp ballot + single-pass decoupled look-back across tiles) and the compaction of
//           every fixed-width column happen in one kernel; the mask never exists in memory.
#include "vm.cuh"

namespace b2 {

constexpr int MAX_TABLE_COLS = 64;

struct OutCols {
  void* data[VM_MAX_OUTS];
  uint32_t* valid[VM_MAX_OUTS];
};

// ------------------------------------------------------------------------------------------------
// project
template <typename T>
__device__ __forceinline__ void store_out(const VMCtx& cx, const Opnd& o, T* __restrict__ out, uint32_t* __restrict__ ovalid) {
  for (int j = 0; j < cx.K; j++) {
    const int i = threadIdx.x + j * VM_NT;
    const int64_t g = cx.tile_base + i;
    const bool in = g < cx.nrows;
    bool v = false;
    if (in) {
      out[g] = opnd_ld<T>(o, i);
      v = opnd_valid(o, i, g);
    }
    if (ovalid) {
      uint32_t bits = __ballot_sync(0xffffffffu, v);
      if ((threadIdx.x & 31) == 0 && in) ovalid[g >> 5] = bits;
    }
  }
}

__global__ void __launch_bounds__(VM_NT, 4) project_kernel(const VMProgramHeader* __restrict__ g_hdr,
                                                        const VMInstr* __restrict__ g_code,
                                                        const __grid_constant__ VMInputs in,
                                                        const __grid_constant__ OutCols outs, int64_t nrows) {
  __shared__ VMShared sh;
  extern __shared__ __align__(16) char regs[];
  const RInstr* code = vm_load_program(sh, g_hdr, g_code, in, regs);
  const int64_t ntiles = (nrows + sh.hdr.tile_rows - 1) / sh.hdr.tile_rows;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    VMCtx cx = vm_ctx(&sh.hdr, &in, regs, tile, nrows);
    vm_run(tile_info(cx), code, 0, sh.hdr.ninstr);
    for (int o = 0; o < sh.hdr.nouts; o++) {
      if (!outs.data[o]) continue;   // a bound reference: the input column itself is the output (refcount bump on the host)
      const int mt = sh.hdr.out_mt[o];
      Opnd op = resolve(cx, sh.hdr.outs[o], mt_width(mt));
      switch (mt_width(mt)) {
        case 1: store_out<int8_t>(cx, op, (int8_t*)outs.data[o], outs.valid[o]); break;
        case 2: store_out<int16_t>(cx, op, (int16_t*)outs.data[o], outs.valid[o]); break;
        case 4: store_out<int32_t>(cx, op, (int32_t*)outs.data[o], outs.valid[o]); break;
        case 8: store_out<int64_t>(cx, op, (int64_t*)outs.data[o], outs.valid[o]); break;
        default: store_out<int4>(cx, op, (int4*)outs.data[o], outs.valid[o]); break;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// ordered single-pass compaction support: decoupled look-back over per-tile counts
constexpr uint64_t LB_AGG = 1ull << 62, LB_PREFIX = 2ull << 62, LB_MASK = (1ull << 62) - 1;

__device__ __forceinline__ uint64_t ld_volatile_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_volatile_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// called by warp 0 of the CTA; returns the number of selected rows in all earlier tiles
__device__ __forceinline__ int64_t lookback_exclusive(uint64_t* status, int64_t tile, uint32_t count) {
  const int lane = threadIdx.x & 31;
  if (tile == 0) {
    if (lane == 0) { __threadfence(); st_volatile_u64(&status[0], LB_PREFIX | count); }
    return 0;
  }
  if (lane == 0) { __threadfence(); st_volatile_u64(&status[tile], LB_AGG | count); }
  int64_t excl = 0;
  int64_t look = tile - 1;
  while (true) {
    const int64_t idx = look - lane;
    uint64_t v;
    if (idx >= 0) {
      do { v = ld_volatile_u64(&status[idx]); } while ((v >> 62) == 0);
    } else {
      v = LB_PREFIX;  // virtual tile before the first one: inclusive prefix 0
    }
    const uint32_t is_prefix = __ballot_sync(0xffffffffu, (v >> 62) == 2);
    const int first = is_prefix ? __ffs(is_prefix) - 1 : 32;
    int64_t contrib = (lane <= first) ? (int64_t)(v & LB_MASK) : 0;
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
    excl += contrib;
    if (is_prefix) break;
    look -= 32;
  }
  if (lane == 0) { __threadfence(); st_volatile_u64(&status[tile], LB_PREFIX | (uint64_t)(excl + count)); }
  return excl;
}

struct FilterCols {
  int32_t ncols;
  int32_t width[MAX_TABLE_COLS];
  const void* in[MAX_TABLE_COLS];
  const uint32_t* in_valid[MAX_TABLE_COLS];
  void* out[MAX_TABLE_COLS];
  uint32_t* out_valid[MAX_TABLE_COLS];  // zero-initialised when present
  int32_t* row_ids;                     // optional gather map of the selected rows (for string columns)
};

struct FilterWork {
  unsigned long long tile_counter;
  unsigned long long total;
};

template <typename T>
__device__ __forceinline__ void compact_one(const void* in, void* out, int64_t g, int64_t pos) {
  reinterpret_cast<T*>(out)[pos] = reinterpret_cast<const T*>(in)[g];
}

// COUNT_ONLY: basicPhysicalOperators.scala:1161-1169 (zero-column batch: just count the trues)
template <bool COUNT_ONLY>
__global__ void __launch_bounds__(VM_NT, 4) filter_kernel(const VMProgramHeader* __restrict__ g_hdr,
                                                       const VMInstr* __restrict__ g_code,
                                                       const __grid_constant__ VMInputs in,
                                                       const __grid_constant__ FilterCols fc, int64_t nrows,
                                                       uint64_t* __restrict__ status, FilterWork* __restrict__ work) {
  constexpr int NW = VM_NT / 32;
  __shared__ VMShared sh;
  __shared__ uint32_t s_counts[VM_MAX_K * NW];  // selected rows per (j, warp) slice, then exclusive offsets
  __shared__ int64_t s_tile_excl;
  __shared__ int64_t s_tile;
  __shared__ uint32_t s_tile_total;
  extern __shared__ __align__(16) char regs[];
  const RInstr* code = vm_load_program(sh, g_hdr, g_code, in, regs);
  const int64_t ntiles = (nrows + sh.hdr.tile_rows - 1) / sh.hdr.tile_rows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long local_count = 0;

  while (true) {
    // tiles are claimed in launch order so that look-back only waits on tiles already running
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(&work->tile_counter, 1ull);
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;

    VMCtx cx = vm_ctx(&sh.hdr, &in, regs, tile, nrows);
    vm_run(tile_info(cx), code, 0, sh.hdr.ninstr);
    const Opnd p = resolve(cx, sh.hdr.outs[0], 1);
    const int K = cx.K;
    uint32_t selmask = 0;
    for (int j = 0; j < K; j++) {
      const int i = threadIdx.x + j * VM_NT;
      const int64_t g = cx.tile_base + i;
      // a NULL predicate drops the row (basicPhysicalOperators.scala:1198-1224)
      const bool sel = g < nrows && opnd_valid(p, i, g) && opnd_ld<int8_t>(p, i) != 0;
      selmask |= (uint32_t)sel << j;
      const uint32_t b = __ballot_sync(0xffffffffu, sel);
      if (lane == 0) s_counts[j * NW + warp] = __popc(b);
    }
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the K*NW slices in row order (4 consecutive slices per lane)
      const int n = K * NW;
      uint32_t c[4], sum = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) { const int e = lane * 4 + k; c[k] = e < n ? s_counts[e] : 0; sum += c[k]; }
      uint32_t inc = sum;
      for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      uint32_t run = inc - sum;
#pragma unroll
      for (int k = 0; k < 4; k++) { const int e = lane * 4 + k; if (e < n) s_counts[e] = run; run += c[k]; }
      const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
      if (COUNT_ONLY) {
        if (lane == 0) local_count += total;
      } else {
        int64_t excl = lookback_exclusive(status, tile, total);
        if (lane == 0) { s_tile_excl = excl; s_tile_total = total; }
      }
    }
    __syncthreads();
    if (!COUNT_ONLY) {
      const int64_t base = s_tile_excl;
      for (int j = 0; j < K; j++) {
        const bool sel = (selmask >> j) & 1u;
        const uint32_t b = __ballot_sync(0xffffffffu, sel);
        if (!sel) continue;
        const int64_t g = cx.tile_base + threadIdx.x + j * VM_NT;
        const int64_t pos = base + s_counts[j * NW + warp] + __popc(b & ((1u << lane) - 1u));
        for (int c = 0; c < fc.ncols; c++) {
          switch (fc.width[c]) {
            case 1: compact_one<int8_t>(fc.in[c], fc.out[c], g, pos); break;
            case 2: compact_one<int16_t>(fc.in[c], fc.out[c], g, pos); break;
            case 4: compact_one<int32_t>(fc.in[c], fc.out[c], g, pos); break;
            case 8: compact_one<int64_t>(fc.in[c], fc.out[c], g, pos); break;
            case 16: compact_one<int4>(fc.in[c], fc.out[c], g, pos); break;
            default: break;  // strings go through the row-id map
          }
          if (fc.out_valid[c] && bit_get(fc.in_valid[c], g)) atomicOr(&fc.out_valid[c][pos >> 5], 1u << (pos & 31));
        }
        if (fc.row_ids) fc.row_ids[pos] = (int32_t)g;
      }
      if (tile == ntiles - 1 && threadIdx.x == 0) work->total = (unsigned long long)(base + s_tile_total);
    }
    __syncthreads();
  }
  if (COUNT_ONLY) {
    if (threadIdx.x == 0 && local_count) atomicAdd(&work->total, local_count);
  }
}


// ---- TMA-staged filter ---------------------------------------------------------------------------------------------------------
// Same contract as filter_kernel<false>, different data movement: every fixed-width column the predicate reads or the
// output keeps is brought into shared memory by TMA bulk copies (cp.async.bulk, one per column and tile, completion on an
// mbarrier).  The whole tile is requested in one go (maximum memory-level parallelism, no load instruction in any row
// loop), the VM reads its column operands from shared memory and the compaction takes the kept values from the same
// staged copy: each input byte crosses HBM exactly once, in large bursts.  Overlap comes from the 3-4 resident CTAs per
// SM being in different phases; a CTA never holds a claimed tile it has not started (a prefetched-but-unstarted tile
// would stall every later tile's look-back for a whole tile time, which made it slower than the direct kernel).
struct FilterStageCols {
  int8_t slot[MAX_TABLE_COLS];   // kept column c -> staged slot (-1: not staged, read from global)
};

__global__ void __launch_bounds__(VM_NT, 4) filter_staged_kernel(const VMProgramHeader* __restrict__ g_hdr, const VMInstr* __restrict__ g_code,
                                                                 const __grid_constant__ VMInputs in, const __grid_constant__ FilterCols fc,
                                                                 const __grid_constant__ VMStage st, const __grid_constant__ FilterStageCols fs,
                                                                 int64_t nrows, uint64_t* __restrict__ status, FilterWork* __restrict__ work) {
  constexpr int NW = VM_NT / 32;
  __shared__ VMShared sh;
  __shared__ uint32_t s_counts[VM_MAX_K * NW];
  __shared__ int64_t s_tile_excl;
  __shared__ int64_t s_tile;
  __shared__ uint32_t s_tile_total;
  __shared__ __align__(8) uint64_t s_bar;
  extern __shared__ __align__(128) char dyn[];
  char* regs = dyn;
  const int R = st.tile_rows;
  const int64_t ntiles = (nrows + R - 1) / R;
  // the stage buffer follows the VM registers (bytes_per_row * R, rounded up to 128 B)
  const int regs_bytes = (g_hdr->bytes_per_row * R + 127) & ~127;
  char* stage = dyn + regs_bytes;
  const RInstr* code = vm_load_program(sh, g_hdr, g_code, in, regs, &st, stage);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
  __syncthreads();
  uint32_t phase = 0;
  while (true) {
    if (threadIdx.x == 0) {
      // tiles are claimed in launch order so that look-back only waits on tiles already being processed
      const int64_t t = (int64_t)atomicAdd(&work->tile_counter, 1ull);
      s_tile = t;
      if (t < ntiles) vm_stage_issue(st, stage, 0, t, nrows, &s_bar);
    }
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) break;
    mbar_wait(&s_bar, phase);   // this tile's columns have landed
    phase ^= 1;
    VMCtx cx = vm_ctx(&sh.hdr, &in, regs, tile, nrows);
    vm_run(tile_info(cx), code, 0, sh.hdr.ninstr);
    const Opnd p = resolve(cx, sh.hdr.outs[0], 1);
    const int K = cx.K;
    uint32_t selmask = 0;
    for (int j = 0; j < K; j++) {
      const int i = threadIdx.x + j * VM_NT;
      const int64_t g = cx.tile_base + i;
      const bool sel = g < nrows && opnd_valid(p, i, g) && opnd_ld<int8_t>(p, i) != 0;
      selmask |= (uint32_t)sel << j;
      const uint32_t b = __ballot_sync(0xffffffffu, sel);
      if (lane == 0) s_counts[j * NW + warp] = __popc(b);
    }
    __syncthreads();
    if (warp == 0) {
      const int n = K * NW;
      uint32_t c[4], sum = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) { const int e = lane * 4 + k; c[k] = e < n ? s_counts[e] : 0; sum += c[k]; }
      uint32_t inc = sum;
      for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      uint32_t run = inc - sum;
#pragma unroll
      for (int k = 0; k < 4; k++) { const int e = lane * 4 + k; if (e < n) s_counts[e] = run; run += c[k]; }
      const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
      int64_t excl = lookback_exclusive(status, tile, total);
      if (lane == 0) { s_tile_excl = excl; s_tile_total = total; }
    }
    __syncthreads();
    const int64_t base = s_tile_excl;
    for (int j = 0; j < K; j++) {
      const bool sel = (selmask >> j) & 1u;
      const uint32_t b = __ballot_sync(0xffffffffu, sel);
      if (!sel) continue;
      const int i = threadIdx.x + j * VM_NT;
      const int64_t g = cx.tile_base + i;
      const int64_t pos = base + s_counts[j * NW + warp] + __popc(b & ((1u << lane) - 1u));
      for (int c = 0; c < fc.ncols; c++) {
        const int sl = fs.slot[c];
        // staged: element i of the tile's copy in shared memory; else straight from global (row g)
        const void* src = sl >= 0 ? (const void*)(stage + st.off[sl]) : fc.in[c];
        const int64_t at = sl >= 0 ? (int64_t)i : g;
        switch (fc.width[c]) {
          case 1: compact_one<int8_t>(src, fc.out[c], at, pos); break;
          case 2: compact_one<int16_t>(src, fc.out[c], at, pos); break;
          case 4: compact_one<int32_t>(src, fc.out[c], at, pos); break;
          case 8: compact_one<int64_t>(src, fc.out[c], at, pos); break;
          case 16: compact_one<int4>(src, fc.out[c], at, pos); break;
          default: break;  // strings go through the row-id map
        }
        if (fc.out_valid[c] && bit_get(fc.in_valid[c], g)) atomicOr(&fc.out_valid[c][pos >> 5], 1u << (pos & 31));
      }
      if (fc.row_ids) fc.row_ids[pos] = (int32_t)g;
    }
    if (tile == ntiles - 1 && threadIdx.x == 0) work->total = (unsigned long long)(base + s_tile_total);
    __syncthreads();   // every reader of the stage buffer is done: the next tile may overwrite it (and s_tile)
  }
}

}  // namespace b2

using namespace b2;

namespace b2 {

void check_program_inputs(const Program* p, const Table* t) {
  if ((int)t->cols.size() < p->hdr.ncols) throw Error(B2_ERR_INVALID, "program references a column the table does not have");
  for (int i = 0; i < p->hdr.ncols; i++) {
    if (p->col_dtype[i] >= 0 && p->col_dtype[i] != t->cols[i]->dtype)
      throw Error(B2_ERR_INVALID, "column " + std::to_string(i) + " has dtype " + std::to_string(t->cols[i]->dtype) +
                                      " but the expression was bound to " + std::to_string(p->col_dtype[i]));
  }
}

void fill_inputs(VMInputs& in, const Table* t) {
  memset(&in, 0, sizeof(in));
  int n = std::min<int>((int)t->cols.size(), VM_MAX_COLS);
  for (int i = 0; i < n; i++) { in.data[i] = t->cols[i]->data.p; in.valid[i] = t->cols[i]->validity(); in.offsets[i] = t->cols[i]->offsets.as<int32_t>(); }
}

int vm_grid(int64_t nrows, int smem_bytes, int tile_rows) {
  int64_t ntiles = (nrows + tile_rows - 1) / tile_rows;
  int per_sm = 8;  // 2048 threads / 256
  int static_smem = (int)sizeof(VMShared) + 1024;
  int by_smem = (227 * 1024) / (smem_bytes + static_smem);
  if (by_smem < per_sm) per_sm = by_smem < 1 ? 1 : by_smem;
  int64_t cap = (int64_t)sm_count() * per_sm;
  return (int)std::max<int64_t>(1, std::min(ntiles, cap));
}

// plan the TMA staging of a filter: every fixed-width column the predicate references or the output keeps
static bool plan_filter_stage(const Program* prog, const Table* pred_table, const FilterCols& fc, const Table* data, VMStage& st, FilterStageCols& fs) {
  memset(&st, 0, sizeof(st));
  memset(st.slot_of_col, -1, sizeof(st.slot_of_col));
  memset(fs.slot, -1, sizeof(fs.slot));
  if (getenv("B2_FILTER_NO_TMA")) return false;
  int bytes_per_row = 0;
  auto add = [&](const Column* c) -> int {
    for (int k = 0; k < st.n; k++) if (st.src[k] == c->data.as<char>()) return k;
    if (st.n >= VM_MAX_STAGED) return -1;
    const int w = dtype_width(c->dtype);
    st.width[st.n] = w; st.src[st.n] = c->data.as<char>(); bytes_per_row += w;
    return st.n++;
  };
  for (int i = 0; i < prog->hdr.ncols && i < (int)pred_table->cols.size(); i++) {
    if (prog->col_dtype[i] < 0 || prog->col_dtype[i] == B2_STRING) continue;   // unreferenced, or read in place by a string predicate
    st.slot_of_col[i] = (int8_t)add(pred_table->cols[i]);
  }
  for (int c = 0; c < fc.ncols; c++) {
    if (fc.width[c] == 0) continue;   // strings travel through the row-id map
    fs.slot[c] = (int8_t)add(data->cols[c]);
  }
  if (st.n == 0 || bytes_per_row == 0) return false;
  // tile: registers + the stage buffer within ~42 KB -> four CTAs per SM, each requesting a whole tile at once
  const int per_row = prog->hdr.bytes_per_row + bytes_per_row;
  int k = (42 * 1024) / (per_row * VM_NT);
  if (k > VM_MAX_K) k = VM_MAX_K;
  if (k < 1) return false;                // rows too wide to stage: the direct kernel handles them
  st.tile_rows = k * VM_NT;
  int off = 0;
  for (int i = 0; i < st.n; i++) { st.off[i] = off; off += st.width[i] * st.tile_rows; }
  st.buf_bytes = (off + 127) & ~127;
  return true;
}

// runs the fused filter; returns the selected-row count.  outputs sized for nrows.
static int64_t run_filter(const Program* prog, const VMInputs& in, FilterCols& fc, int64_t nrows, bool count_only,
                          const Table* pred_table = nullptr, const Table* data = nullptr) {
  if (nrows == 0) return 0;
  DevBuf work(sizeof(FilterWork));
  CUDA_CHECK(cudaMemsetAsync(work.p, 0, sizeof(FilterWork), stream()));
  VMStage st; FilterStageCols fs;
  const bool staged = !count_only && pred_table && data && nrows >= (1 << 16) && plan_filter_stage(prog, pred_table, fc, data, st, fs);
  const int tile_rows = staged ? st.tile_rows : prog->hdr.tile_rows;
  int64_t ntiles = (nrows + tile_rows - 1) / tile_rows;
  DevBuf status;
  if (!count_only) {
    status = DevBuf((size_t)ntiles * 8);
    CUDA_CHECK(cudaMemsetAsync(status.p, 0, (size_t)ntiles * 8, stream()));
  }
  int smem = prog->hdr.smem_bytes;
  int grid = vm_grid(nrows, smem, prog->hdr.tile_rows);
  if (staged) {
    const int regs_bytes = (prog->hdr.bytes_per_row * st.tile_rows + 127) & ~127;
    smem = regs_bytes + st.buf_bytes;
    const int per_sm = std::max(1, std::min(4, (224 * 1024) / (smem + (int)sizeof(VMShared) + 2048)));
    grid = (int)std::max<int64_t>(1, std::min<int64_t>(ntiles, (int64_t)sm_count() * per_sm));
    launch("filter_staged_kernel", filter_staged_kernel, grid, VM_NT, smem, stream(), prog->d_hdr.as<VMProgramHeader>(), prog->d_code.as<VMInstr>(), in, fc,
           st, fs, nrows, status.as<uint64_t>(), work.as<FilterWork>());
  } else if (count_only) {
    launch("filter_count_kernel", filter_kernel<true>, grid, VM_NT, smem, stream(), prog->d_hdr.as<VMProgramHeader>(), prog->d_code.as<VMInstr>(), in, fc,
           nrows, nullptr, work.as<FilterWork>());
  } else {
    launch("filter_kernel", filter_kernel<false>, grid, VM_NT, smem, stream(), prog->d_hdr.as<VMProgramHeader>(), prog->d_code.as<VMInstr>(), in, fc,
           nrows, status.as<uint64_t>(), work.as<FilterWork>());
  }
  FilterWork hw;
  d2h(&hw, work.p, 1);
  sync();
  return (int64_t)hw.total;
}

Table* gather_table(const Table* t, const int32_t* d_map, int64_t n, bool nullify_oob, const std::vector<int>* only_cols);

// shared by b2_filter and b2_filter_mask: `pred_table` feeds the program, `data` is compacted
static Table* filter_impl(const Program* prog, const Table* pred_table, const Table* data) {
  check_program_inputs(prog, pred_table);
  B2_CHECK(prog->hdr.nouts >= 1 && prog->out_dtype[0] == B2_BOOL8, "filter predicate must be a single BOOL8 expression");
  B2_CHECK((int)data->cols.size() <= MAX_TABLE_COLS, "too many columns");
  const int64_t n = data->rows;
  VMInputs in; fill_inputs(in, pred_table);
  FilterCols fc; memset(&fc, 0, sizeof(fc));
  fc.ncols = (int)data->cols.size();
  ColsGuard outs;
  bool has_strings = false;
  for (int c = 0; c < fc.ncols; c++) {
    const Column* ic = data->cols[c];
    if (ic->dtype == B2_STRING) { has_strings = true; outs.v.push_back(nullptr); fc.width[c] = 0; continue; }
    Column* oc = new_column(ic->dtype, ic->scale, n, ic->nullable());
    outs.v.push_back(oc);
    fc.width[c] = dtype_width(ic->dtype);
    fc.in[c] = ic->data.p; fc.in_valid[c] = ic->validity();
    fc.out[c] = oc->data.p; fc.out_valid[c] = oc->valid.as<uint32_t>();
    if (oc->valid.p) CUDA_CHECK(cudaMemsetAsync(oc->valid.p, 0, oc->valid.bytes, stream()));
  }
  DevBuf row_ids;
  if (has_strings) { row_ids = DevBuf((size_t)std::max<int64_t>(n, 1) * 4); fc.row_ids = row_ids.as<int32_t>(); }
  int64_t count = run_filter(prog, in, fc, n, false, pred_table, data);
  // shrink: keep the over-allocated buffers only when most rows survived
  for (int c = 0; c < fc.ncols; c++) {
    Column* oc = outs.v[c];
    if (!oc) continue;
    oc->size = count;
    if (count * 2 < n) {
      int w = dtype_width(oc->dtype);
      DevBuf nd((size_t)count * w);
      if (count) CUDA_CHECK(cudaMemcpyAsync(nd.p, oc->data.p, (size_t)count * w, cudaMemcpyDeviceToDevice, stream()));
      oc->data = std::move(nd);
      if (oc->valid.p) {
        DevBuf nv(validity_bytes(count));
        CUDA_CHECK(cudaMemcpyAsync(nv.p, oc->valid.p, nv.bytes, cudaMemcpyDeviceToDevice, stream()));
        oc->valid = std::move(nv);
      }
    }
    oc->null_count = oc->valid.p ? -1 : 0;
  }
  if (has_strings) {
    std::vector<int> scols;
    for (int c = 0; c < fc.ncols; c++) if (!outs.v[c]) scols.push_back(c);
    Table* st = gather_table(data, row_ids.as<int32_t>(), count, false, &scols);
    for (size_t k = 0; k < scols.size(); k++) { outs.v[scols[k]] = st->cols[k]; st->cols[k] = nullptr; }
    st->cols.clear();
    delete st;
  }
  return new_table(outs.release());
}

}  // namespace b2

namespace b2 {
// GpuFilterExec under a column-pruning GpuProjectExec, fused: the predicate sees the whole batch, only `keep` is compacted
Table* filter_select(const Program* prog, const Table* t, const int32_t* keep, int nkeep) {
  Table view;
  struct Unhook { Table& t; ~Unhook() { t.cols.clear(); } } unhook{view};  // the view does not own its columns
  for (int k = 0; k < nkeep; k++) {
    if (keep[k] < 0 || keep[k] >= (int)t->cols.size()) throw Error(B2_ERR_INVALID, "filter: output column out of range");
    view.cols.push_back(t->cols[keep[k]]);
  }
  view.rows = t->rows;
  return filter_impl(prog, t, &view);
}

// selection vector: the row ids that pass the predicate, in order, and nothing else (late materialisation: a join probe or
// an exchange scatter directly above the filter reads the batch through it instead of through a compacted copy)
bool simple_filter_row_ids(const Program* prog, const Table* t, Column** out);   // simplefilter.cu
Column* filter_row_ids(const Program* prog, const Table* t) {
  check_program_inputs(prog, t);
  B2_CHECK(prog->hdr.nouts >= 1 && prog->out_dtype[0] == B2_BOOL8, "filter predicate must be a single BOOL8 expression");
  const int64_t n = t->rows;
  Column* fast = nullptr;
  if (simple_filter_row_ids(prog, t, &fast)) return fast;   // conjunction of column-vs-literal comparisons: no VM
  VMInputs in; fill_inputs(in, t);
  FilterCols fc; memset(&fc, 0, sizeof(fc));
  ColGuard ids(new_column(B2_INT32, 0, n, false));
  fc.row_ids = ids.c->data.as<int32_t>();
  Table none;   // no payload columns: only the predicate's inputs are staged
  ids.c->size = run_filter(prog, in, fc, n, false, t, &none);
  return ids.release();
}

// Table.filter(mask): order-preserving compaction of every column by a BOOL8 mask (NULL = drop)
Table* filter_by_mask(const Table* t, Column* m) {
  B2_CHECK(m->dtype == B2_BOOL8, "filter mask must be BOOL8");
  B2_CHECK(m->size == t->rows, "mask length differs from the table");
  // a zero-instruction program whose single output is input column 0 (the mask)
  Program prog; memset(&prog.hdr, 0, sizeof(prog.hdr));
  prog.hdr.nouts = 1; prog.hdr.ncols = 1;
  prog.hdr.outs[0].kind = OK_COL; prog.hdr.outs[0].idx = 0; prog.hdr.outs[0].nullable = 1;
  prog.hdr.out_mt[0] = MT_I8;
  set_tile_geometry(prog.hdr, 0);
  prog.col_dtype = {B2_BOOL8};
  prog.out_dtype = {B2_BOOL8}; prog.out_scale = {0}; prog.out_precision = {0}; prog.out_nullable = {1};
  prog.d_hdr = DevBuf(sizeof(VMProgramHeader));
  h2d(prog.d_hdr.p, &prog.hdr, 1);
  prog.d_code = DevBuf(sizeof(VMInstr));
  Table mt; mt.cols = {m}; mt.rows = m->size;
  struct Unhook { Table& t; ~Unhook() { t.cols.clear(); } } unhook{mt};  // mt does not own m
  return filter_impl(&prog, &mt, t);
}

}  // namespace b2

extern "C" {

int b2_project(b2_handle program, b2_handle table, b2_handle* out_table) {
  B2_TRY
  Program* prog = program_from(program);
  Table* t = table_from(table);
  check_program_inputs(prog, t);
  const int64_t n = t->rows;
  VMInputs in; fill_inputs(in, t);
  OutCols oc; memset(&oc, 0, sizeof(oc));
  ColsGuard outs;
  int computed = 0;
  for (int o = 0; o < prog->hdr.nouts; o++) {
    const VMOperand& op = prog->hdr.outs[o];
    if (op.kind == OK_COL) {
      // GpuBoundReference.columnarEval: the output IS the input column, by refcount (basicPhysicalOperators.scala:117-119
      // "no-op project just bumps refcounts"); also the only way a STRING column passes through a projection
      Column* c = t->cols[op.idx];
      col_incref(c);
      outs.v.push_back(c);
      continue;
    }
    if (prog->out_dtype[o] == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "computed string outputs (use b2_substring for Substring)");
    Column* c = new_column(prog->out_dtype[o], prog->out_scale[o], n, prog->out_nullable[o]);
    outs.v.push_back(c);
    oc.data[o] = c->data.p; oc.valid[o] = c->valid.as<uint32_t>();
    computed++;
  }
  if (n > 0 && computed > 0) {
    const int smem = prog->hdr.smem_bytes;
    launch("project_kernel", project_kernel, vm_grid(n, smem, prog->hdr.tile_rows), VM_NT, smem, stream(), prog->d_hdr.as<VMProgramHeader>(),
           prog->d_code.as<VMInstr>(), in, oc, n);
  }
  *out_table = to_handle(new_table(outs.release()));
  B2_CATCH
}

int b2_filter(b2_handle predicate_program, b2_handle table, b2_handle* out_table) {
  B2_TRY
  Table* t = table_from(table);
  *out_table = to_handle(filter_impl(program_from(predicate_program), t, t));
  B2_CATCH
}

int b2_filter_select(b2_handle predicate_program, b2_handle table, const int32_t* keep_cols, int32_t nkeep, b2_handle* out_table) {
  B2_TRY
  *out_table = to_handle(filter_select(program_from(predicate_program), table_from(table), keep_cols, nkeep));
  B2_CATCH
}

int b2_filter_row_ids(b2_handle predicate_program, b2_handle table, b2_handle* out_int32_ids) {
  B2_TRY
  *out_int32_ids = to_handle(filter_row_ids(program_from(predicate_program), table_from(table)));
  B2_CATCH
}

int b2_filter_count(b2_handle predicate_program, b2_handle table, int64_t* out_count) {
  B2_TRY
  Program* prog = program_from(predicate_program);
  Table* t = table_from(table);
  check_program_inputs(prog, t);
  B2_CHECK(prog->hdr.nouts >= 1 && prog->out_dtype[0] == B2_BOOL8, "filter predicate must be a single BOOL8 expression");
  VMInputs in; fill_inputs(in, t);
  FilterCols fc; memset(&fc, 0, sizeof(fc));
  *out_count = run_filter(prog, in, fc, t->rows, true);
  B2_CATCH
}

int b2_filter_mask(b2_handle table, b2_handle bool_mask, b2_handle* out_table) {
  B2_TRY
  *out_table = to_handle(filter_by_mask(table_from(table), col_from(bool_mask)));
  B2_CATCH
}

}  // extern "C"
