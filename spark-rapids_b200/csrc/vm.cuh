// vm.cuh — the fused expression evaluator: a register machine whose registers are typed column
// slices in shared memory.  One CTA owns a tile of hdr.tile_rows rows; thread t owns rows
// t + j*VM_NT (j < K), so every register access is thread-private (no barriers between
// instructions) and bank-conflict free, while every global column access is fully coalesced (a warp
// reads 32 consecutive rows).  The tile is sized per program (as many rows as fit ~40 KB of
// registers) so that one instruction dispatch — and one trip through the instruction cache — is
// amortised over thousands of rows: a vectorised interpreter, with vectors living in shared memory.
//
// Replaces the reference's one-cudf-kernel-per-expression-node evaluation with full intermediate
// columns (GpuExpressions.scala:397-413 CudfBinaryExpression.doColumnar; SURVEY §8a a1): here the
// whole bound expression list of a GpuProjectExec / GpuFilterExec / aggregate pre-step is ONE
// kernel, intermediates never leave the SM.
#pragma once
#include "common.cuh"

namespace b2 {

constexpr int VM_NT = 256;           // threads per CTA
constexpr int VM_MAX_K = 16;         // rows per thread per tile (tile_rows = K * VM_NT <= 4096)
constexpr int VM_SMEM_BUDGET = 40 * 1024;        // register bytes per tile (narrow programs: 4 CTAs/SM)
constexpr int VM_SMEM_BUDGET_WIDE = 72 * 1024;   // programs with wide rows (>= 24 B/row of registers): 2 CTAs/SM, more rows per dispatch
constexpr int VM_MAX_REGS = 64;
constexpr int VM_MAX_COLS = 64;
constexpr int VM_MAX_OUTS = 32;

enum MT : uint8_t { MT_I8 = 0, MT_I16 = 1, MT_I32 = 2, MT_I64 = 3, MT_I128 = 4, MT_F32 = 5, MT_F64 = 6 };
__host__ __device__ inline int mt_width(int mt) {
  switch (mt) { case MT_I8: return 1; case MT_I16: return 2; case MT_I32: case MT_F32: return 4;
                case MT_I64: case MT_F64: return 8; default: return 16; }
}

enum OK : uint8_t { OK_NONE = 0, OK_REG = 1, OK_COL = 2, OK_LIT = 3 };

enum VOP : uint8_t {
  V_ADD = 1, V_SUB, V_MUL, V_DIV, V_MOD, V_PMOD, V_NEG, V_ABS,
  V_EQ, V_NE, V_LT, V_LE, V_GT, V_GE, V_EQNS,
  V_AND, V_OR, V_NOT,
  V_ISNULL, V_ISNOTNULL, V_COALESCE, V_IF,
  V_CAST,        // mt = source, mt2 = destination machine type
  V_RESCALE_UP,  // integer * 10^aux with overflow -> null (decimal scale increase); mt=mt2 width
  V_RESCALE_DOWN,// integer / 10^aux HALF_UP (decimal scale decrease)
  V_CHECK_PREC,  // |x| >= 10^aux -> null  (CheckOverflow / GpuCheckOverflow)
  V_MULW,        // widening multiply: two I64 operands -> exact I128 product
  V_DIVDEC,      // decimal divide: round_half_up(a * 10^aux / b), b == 0 or > 38 digits -> null
  V_MULDEC,      // 128x128 -> 256-bit product, / 10^aux HALF_UP, overflow -> null
  V_DEC2F64,     // decimal (mt) -> double, / 10^aux
  V_NORM_NAN_ZERO,
  V_YEAR,
  V_MOV,
  V_ANDCMP,     // c AND (a <cmp> b), all operands non-null: aux = 3-bit truth mask over sign(a ? b) = {<, ==, >}
  V_STRPRED     // string predicate -> BOOL8.  a = STRING column, b = STRING column or pooled literal (mt2 = 1), c = optional
                // substring window literal (lo = pos, hi = len; Spark 1-based substringSQL) applied to a;
                // aux = kind (SP_*) | escape char << 8 (LIKE)
};
// stringFunctions.scala:163 GpuStartsWith, :189 GpuEndsWith, :396 GpuContains, :972 GpuLike; predicates.scala:155-331 on strings
// (UTF8String.compareTo = unsigned byte order)
enum SPK : int { SP_EQ = 0, SP_NE, SP_LT, SP_LE, SP_GT, SP_GE, SP_STARTS, SP_ENDS, SP_CONTAINS, SP_LIKE };
constexpr int VM_LIT_BYTES = 512;   // pooled string literals of a program

struct alignas(16) VMOperand {
  int64_t lo, hi;    // OK_LIT value (first so that 16-byte literal loads are aligned)
  int32_t idx;       // register or input column index
  uint8_t kind;      // OK
  uint8_t nullable;  // may carry nulls
  uint8_t lit_null;  // OK_LIT: literal is NULL
  uint8_t pad;
};

struct alignas(16) VMInstr {
  uint8_t op, mt, mt2, dst_nullable;
  int32_t dst;
  int32_t aux;
  int32_t pad;
  VMOperand a, b, c;
};

struct VMReg { int32_t off; int32_t voff; };  // offsets in BYTES PER ROW (x tile_rows = bytes inside the tile)

struct VMProgramHeader {
  int32_t ninstr, nregs, ncols, nouts;
  int32_t smem_bytes;   // = bytes_per_row * tile_rows
  int32_t bytes_per_row, tile_rows, npred;  // npred: leading instructions that compute output 0 (the predicate)
  VMReg regs[VM_MAX_REGS];
  VMOperand outs[VM_MAX_OUTS];
  uint8_t out_mt[VM_MAX_OUTS];
  char lits[VM_LIT_BYTES];   // string literal pool (OK_LIT string operand: lo = offset, hi = length)
};

struct VMInputs {
  const void* data[VM_MAX_COLS];
  const uint32_t* valid[VM_MAX_COLS];
  const int32_t* offsets[VM_MAX_COLS];   // STRING columns
};

// instruction with operands resolved once per CTA (shared memory): a row loop starts with two
// 16-byte shared loads per operand instead of re-deriving pointers from the program header
struct alignas(16) ROpnd {
  const char* base;      // tile-0 address: register slice (shared), column data (global) or literal
  const void* vptr;      // validity bytes (shared) or bitmask (global)
  int32_t stride;        // bytes per row, 0 for a literal
  int32_t tile_step;     // bytes per row to advance per tile row offset (columns only)
  int32_t vkind;         // 0 valid, 1 bytes, 2 bitmask, 3 null
  int32_t pad;
};
struct alignas(16) RInstr {
  uint8_t op, mt, mt2, dst_nullable;
  int32_t aux;
  char* dbase;
  uint8_t* dvb;
  int64_t pad;
  ROpnd a, b, c;
};

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------

__device__ __forceinline__ i128 pow10_i128(int e) {
  // 10^e for 0 <= e <= 38
  const unsigned long long p19 = 10000000000000000000ull;  // 10^19
  unsigned long long small = 1;
  int r = e >= 19 ? e - 19 : e;
  for (int i = 0; i < r; i++) small *= 10ull;
  return e >= 19 ? (i128)((u128)small * (u128)p19) : (i128)small;
}

// resolved per instruction, uniform across the CTA
struct Opnd {
  const char* base;  // generic pointer: shared register slice, global column (pre-offset to tile) or literal
  int stride;        // bytes per row (0 for a literal)
  int vkind;         // 0 always valid, 1 byte-per-row (shared), 2 bitmask (global), 3 always null
  const uint8_t* vbytes;
  const uint32_t* vbits;
};

struct VMCtx {
  const VMProgramHeader* hdr;
  const VMInputs* in;
  char* smem;
  int64_t tile_base;  // first global row of this tile
  int64_t nrows;
  int K;              // rows per thread in this tile
  int tile_rows;
  uint32_t rowmask;   // bit j set = this thread's row j is wanted (post-predicate instructions)
  int stage_off;      // staged input columns (TMA double buffer): byte offset of the buffer holding this tile
};

__device__ __forceinline__ Opnd resolve(const VMCtx& cx, const VMOperand& o, int width) {
  Opnd r;
  r.vbytes = nullptr; r.vbits = nullptr;
  if (o.kind == OK_REG) {
    r.base = cx.smem + (size_t)cx.hdr->regs[o.idx].off * cx.tile_rows;
    r.stride = width;
    r.vkind = o.nullable ? 1 : 0;
    r.vbytes = reinterpret_cast<const uint8_t*>(cx.smem + (size_t)cx.hdr->regs[o.idx].voff * cx.tile_rows);
  } else if (o.kind == OK_COL) {
    r.base = reinterpret_cast<const char*>(cx.in->data[o.idx]) + cx.tile_base * width;
    r.stride = width;
    const uint32_t* vb = cx.in->valid[o.idx];
    r.vkind = (o.nullable && vb) ? 2 : 0;
    r.vbits = vb;
  } else {
    r.base = reinterpret_cast<const char*>(&o.lo);
    r.stride = 0;
    r.vkind = o.lit_null ? 3 : 0;
  }
  return r;
}

template <typename T>
__device__ __forceinline__ T opnd_ld(const Opnd& o, int i) {
  return *reinterpret_cast<const T*>(o.base + (size_t)i * o.stride);
}
__device__ __forceinline__ bool opnd_valid(const Opnd& o, int i, int64_t g) {
  switch (o.vkind) {
    case 0: return true;
    case 1: return o.vbytes[i] != 0;
    case 2: return bit_get(o.vbits, g);
    default: return false;
  }
}

struct Dst {
  char* base; int stride; uint8_t* vbytes; bool nullable;
};
__device__ __forceinline__ Dst resolve_dst(const VMCtx& cx, const VMInstr& ins, int width) {
  Dst d;
  d.base = cx.smem + (size_t)cx.hdr->regs[ins.dst].off * cx.tile_rows;
  d.stride = width;
  d.vbytes = reinterpret_cast<uint8_t*>(cx.smem + (size_t)cx.hdr->regs[ins.dst].voff * cx.tile_rows);
  d.nullable = ins.dst_nullable;
  return d;
}
template <typename T>
__device__ __forceinline__ void dst_st(const Dst& d, int i, T v, bool valid) {
  *reinterpret_cast<T*>(d.base + (size_t)i * d.stride) = v;
  if (d.nullable) d.vbytes[i] = valid ? 1 : 0;
}

template <typename T> struct UnsignedOf { typedef T type; };
template <> struct UnsignedOf<int8_t> { typedef uint8_t type; };
template <> struct UnsignedOf<int16_t> { typedef uint16_t type; };
template <> struct UnsignedOf<int32_t> { typedef uint32_t type; };
template <> struct UnsignedOf<int64_t> { typedef uint64_t type; };
template <> struct UnsignedOf<i128> { typedef u128 type; };
template <typename T> struct IsFloat { static const bool v = false; };
template <> struct IsFloat<float> { static const bool v = true; };
template <> struct IsFloat<double> { static const bool v = true; };

// row loops.  Rows are processed in batches of VM_B: all operand loads of a batch are issued before
// any store (registers may alias: a destination slot can recycle a source slot), which also keeps
// VM_B independent loads in flight per thread.
constexpr int VM_B = 4;  // the VM_LD*/VM_ST* expansions below are written for exactly 4
// The context lives in the caller's frame (local memory) and every store through a register
// pointer could alias it, so handlers copy what the row loops need into registers ONCE.
struct TileInfo { int K; uint32_t rowmask; int64_t tile_base, nrows; int tile_rows; int stage_off; };
__device__ __forceinline__ TileInfo tile_info(const VMCtx& cx) {
  TileInfo t; t.K = cx.K; t.rowmask = cx.rowmask; t.tile_base = cx.tile_base; t.nrows = cx.nrows; t.tile_rows = cx.tile_rows; t.stage_off = cx.stage_off; return t;
}
__device__ __forceinline__ Opnd ropnd(const ROpnd& o, const TileInfo& ti) {
  Opnd r;
  r.base = o.base + ti.tile_base * o.tile_step + (o.pad ? ti.stage_off : 0);   // pad = 1: a column staged in shared memory by TMA
  r.stride = o.stride; r.vkind = o.vkind;
  r.vbytes = reinterpret_cast<const uint8_t*>(o.vptr); r.vbits = reinterpret_cast<const uint32_t*>(o.vptr);
  return r;
}
__device__ __forceinline__ Dst rdst(const RInstr& ins, int width) {
  Dst d; d.base = ins.dbase; d.stride = width; d.vbytes = ins.dvb; d.nullable = ins.dst_nullable; return d;
}
#define VM_ROW_ACTIVE(j, i, g) \
  const int i = threadIdx.x + (j) * VM_NT; const int64_t g = ti.tile_base + i; \
  const bool act = (j) < ti.K && g < ti.nrows && ((ti.rowmask >> (j)) & 1u)

// Row loops come in two flavours, chosen once per instruction (uniformly for the CTA):
//   fast    : full tile, every row wanted, no operand carries NULLs and the result cannot be NULL.
//             Per-thread base pointers + compile-time offsets: a row costs its loads, the ALU op and
//             one store.  Literals are read once, outside the loop.
//   checked : everything else (last tile, post-predicate row mask, NULL propagation).
// Both issue all loads of a 4-row batch before any store (a destination slot may recycle a source
// slot) and keep the batch in named scalars — indexed arrays ended up in local memory.
__device__ __forceinline__ bool vm_full_tile(const TileInfo& ti, int tile_rows) {
  return ti.tile_base + tile_rows <= ti.nrows && ti.rowmask == 0xffffffffu;
}
template <typename T>
__device__ __forceinline__ const char* thread_base(const Opnd& o) { return o.base + (size_t)threadIdx.x * o.stride; }

#define VM_LD1(u)                                                                              \
  const int i##u = threadIdx.x + (j0 + u) * VM_NT; const int64_t g##u = ti.tile_base + i##u;    \
  const bool act##u = (j0 + u) < ti.K && g##u < ti.nrows && ((ti.rowmask >> (j0 + u)) & 1u);  \
  T x##u = T(); bool v##u = false;                                                             \
  if (act##u) { x##u = opnd_ld<T>(a, i##u); v##u = opnd_valid(a, i##u, g##u); }
#define VM_ST1(u) if (act##u) { bool vv = v##u; const R r = f(x##u, vv); dst_st<R>(d, i##u, r, vv); }
#define VM_LD2(u)                                                                              \
  const int i##u = threadIdx.x + (j0 + u) * VM_NT; const int64_t g##u = ti.tile_base + i##u;    \
  const bool act##u = (j0 + u) < ti.K && g##u < ti.nrows && ((ti.rowmask >> (j0 + u)) & 1u);  \
  T x##u = T(); TB y##u = TB(); bool va##u = false, vb##u = false;                             \
  if (act##u) { x##u = opnd_ld<T>(a, i##u); y##u = opnd_ld<TB>(b, i##u); va##u = opnd_valid(a, i##u, g##u); vb##u = opnd_valid(b, i##u, g##u); }
#define VM_ST2(u) if (act##u) { bool vv = va##u && vb##u; const R r = f(x##u, y##u, va##u, vb##u, vv); dst_st<R>(d, i##u, r, vv); }

// unary: F(T x, bool& valid) -> R
template <typename T, typename R, typename F>
__device__ __forceinline__ void vm_loop1(const TileInfo ti, const RInstr& ins, F f) {
  const Opnd a = ropnd(ins.a, ti);
  const Dst d = rdst(ins, sizeof(R));
  if (a.vkind == 0 && !d.nullable && a.stride != 0 && vm_full_tile(ti, ti.tile_rows)) {
    const char* pa = thread_base<T>(a);
    char* pd = d.base + (size_t)threadIdx.x * sizeof(R);
    for (int j0 = 0; j0 + 4 <= ti.K; j0 += 4, pa += 4 * VM_NT * sizeof(T), pd += 4 * VM_NT * sizeof(R)) {
      const T x0 = *reinterpret_cast<const T*>(pa), x1 = *reinterpret_cast<const T*>(pa + VM_NT * sizeof(T)),
              x2 = *reinterpret_cast<const T*>(pa + 2 * VM_NT * sizeof(T)), x3 = *reinterpret_cast<const T*>(pa + 3 * VM_NT * sizeof(T));
      bool vv = true;
      *reinterpret_cast<R*>(pd) = f(x0, vv); *reinterpret_cast<R*>(pd + VM_NT * sizeof(R)) = f(x1, vv);
      *reinterpret_cast<R*>(pd + 2 * VM_NT * sizeof(R)) = f(x2, vv); *reinterpret_cast<R*>(pd + 3 * VM_NT * sizeof(R)) = f(x3, vv);
    }
    for (int j = ti.K & ~3; j < ti.K; j++, pa += VM_NT * sizeof(T), pd += VM_NT * sizeof(R)) {
      bool vv = true;
      *reinterpret_cast<R*>(pd) = f(*reinterpret_cast<const T*>(pa), vv);
    }
    return;
  }
  for (int j0 = 0; j0 < ti.K; j0 += VM_B) {
    VM_LD1(0) VM_LD1(1) VM_LD1(2) VM_LD1(3)
    VM_ST1(0) VM_ST1(1) VM_ST1(2) VM_ST1(3)
  }
}
// binary: F(T x, TB y, bool va, bool vb, bool& valid) -> R
template <typename T, typename R, typename TB, typename F>
__device__ __forceinline__ void vm_loop2x(const TileInfo ti, const RInstr& ins, F f) {
  const Opnd a = ropnd(ins.a, ti), b = ropnd(ins.b, ti);
  const Dst d = rdst(ins, sizeof(R));
  if (a.vkind == 0 && b.vkind == 0 && !d.nullable && a.stride != 0 && vm_full_tile(ti, ti.tile_rows)) {
    const char* pa = thread_base<T>(a);
    char* pd = d.base + (size_t)threadIdx.x * sizeof(R);
    bool vv = true;
    if (b.stride == 0) {  // column/register (op) literal
      const TB y = *reinterpret_cast<const TB*>(b.base);
      int j0 = 0;
      if constexpr (sizeof(T) <= 8 && sizeof(R) <= 8) {
        for (; j0 + 8 <= ti.K; j0 += 8, pa += 8 * VM_NT * sizeof(T), pd += 8 * VM_NT * sizeof(R)) {
          T x[8];
#pragma unroll
          for (int u = 0; u < 8; u++) x[u] = *reinterpret_cast<const T*>(pa + u * VM_NT * sizeof(T));
#pragma unroll
          for (int u = 0; u < 8; u++) *reinterpret_cast<R*>(pd + u * VM_NT * sizeof(R)) = f(x[u], y, true, true, vv);
        }
      }
      for (; j0 + 4 <= ti.K; j0 += 4, pa += 4 * VM_NT * sizeof(T), pd += 4 * VM_NT * sizeof(R)) {
        const T x0 = *reinterpret_cast<const T*>(pa), x1 = *reinterpret_cast<const T*>(pa + VM_NT * sizeof(T)),
                x2 = *reinterpret_cast<const T*>(pa + 2 * VM_NT * sizeof(T)), x3 = *reinterpret_cast<const T*>(pa + 3 * VM_NT * sizeof(T));
        *reinterpret_cast<R*>(pd) = f(x0, y, true, true, vv); *reinterpret_cast<R*>(pd + VM_NT * sizeof(R)) = f(x1, y, true, true, vv);
        *reinterpret_cast<R*>(pd + 2 * VM_NT * sizeof(R)) = f(x2, y, true, true, vv); *reinterpret_cast<R*>(pd + 3 * VM_NT * sizeof(R)) = f(x3, y, true, true, vv);
      }
      for (; j0 < ti.K; j0++, pa += VM_NT * sizeof(T), pd += VM_NT * sizeof(R))
        *reinterpret_cast<R*>(pd) = f(*reinterpret_cast<const T*>(pa), y, true, true, vv);
    } else {
      const char* pb = thread_base<TB>(b);
      for (int j0 = 0; j0 + 4 <= ti.K; j0 += 4, pa += 4 * VM_NT * sizeof(T), pb += 4 * VM_NT * sizeof(TB), pd += 4 * VM_NT * sizeof(R)) {
        const T x0 = *reinterpret_cast<const T*>(pa), x1 = *reinterpret_cast<const T*>(pa + VM_NT * sizeof(T)),
                x2 = *reinterpret_cast<const T*>(pa + 2 * VM_NT * sizeof(T)), x3 = *reinterpret_cast<const T*>(pa + 3 * VM_NT * sizeof(T));
        const TB y0 = *reinterpret_cast<const TB*>(pb), y1 = *reinterpret_cast<const TB*>(pb + VM_NT * sizeof(TB)),
                 y2 = *reinterpret_cast<const TB*>(pb + 2 * VM_NT * sizeof(TB)), y3 = *reinterpret_cast<const TB*>(pb + 3 * VM_NT * sizeof(TB));
        *reinterpret_cast<R*>(pd) = f(x0, y0, true, true, vv); *reinterpret_cast<R*>(pd + VM_NT * sizeof(R)) = f(x1, y1, true, true, vv);
        *reinterpret_cast<R*>(pd + 2 * VM_NT * sizeof(R)) = f(x2, y2, true, true, vv); *reinterpret_cast<R*>(pd + 3 * VM_NT * sizeof(R)) = f(x3, y3, true, true, vv);
      }
      for (int j = ti.K & ~3; j < ti.K; j++, pa += VM_NT * sizeof(T), pb += VM_NT * sizeof(TB), pd += VM_NT * sizeof(R))
        *reinterpret_cast<R*>(pd) = f(*reinterpret_cast<const T*>(pa), *reinterpret_cast<const TB*>(pb), true, true, vv);
    }
    return;
  }
  for (int j0 = 0; j0 < ti.K; j0 += VM_B) {
    VM_LD2(0) VM_LD2(1) VM_LD2(2) VM_LD2(3)
    VM_ST2(0) VM_ST2(1) VM_ST2(2) VM_ST2(3)
  }
}

template <typename T, typename R, typename F>
__device__ __forceinline__ void vm_loop2(const TileInfo ti, const RInstr& ins, F f) { vm_loop2x<T, R, T>(ti, ins, f); }

// Spark comparison semantics (predicates.scala:155-331): NaN == NaN, NaN greater than all, -0.0 == 0.0
template <typename T>
__device__ __forceinline__ int cmp3(T a, T b) {
  if constexpr (IsFloat<T>::v) {
    bool an = a != a, bn = b != b;
    if (an || bn) return an == bn ? 0 : (an ? 1 : -1);
  }
  return a < b ? -1 : (a > b ? 1 : 0);
}

template <typename T, int OP>
__device__ __noinline__ void vm_arith(const TileInfo ti, const RInstr& ins) {
  typedef typename UnsignedOf<T>::type U;
  vm_loop2<T, T>(ti, ins, [](T x, T y, bool, bool, bool& v) -> T {
    if constexpr (IsFloat<T>::v) {
      // arithmetic.scala:309-340 — IEEE; Divide/Remainder by zero -> NULL (Spark non-ANSI)
      if constexpr (OP == V_ADD) return x + y;
      else if constexpr (OP == V_SUB) return x - y;
      else if constexpr (OP == V_MUL) return x * y;
      else if constexpr (OP == V_DIV) { if (y == (T)0) { v = false; return (T)0; } return x / y; }
      else {
        if (y == (T)0) { v = false; return (T)0; }
        T r = (T)fmod((double)x, (double)y);
        // Spark Pmod / cudf BinaryOp.PMOD (arithmetic.scala:1177): r = a % n; if (r < 0) (r + n) % n else r
        if (OP == V_PMOD && r < (T)0) r = (T)fmod((double)(r + y), (double)y);
        return r;
      }
    } else {
      // integer: two's-complement wrap (arithmetic.scala:38-75, non-ANSI)
      if constexpr (OP == V_ADD) return (T)((U)x + (U)y);
      else if constexpr (OP == V_SUB) return (T)((U)x - (U)y);
      else if constexpr (OP == V_MUL) return (T)((U)x * (U)y);
      else {
        if (y == (T)0) { v = false; return (T)0; }
        if (y == (T)-1) return (OP == V_DIV) ? (T)((U)0 - (U)x) : (T)0;
        if constexpr (OP == V_DIV) return x / y;
        else {
          T r = x % y;
          if (OP == V_PMOD && r < 0) {  // (r + n) % n with Java's wrap-around add in the operand type (byte/short add in int)
            if constexpr (sizeof(T) < 4) r = (T)(((int)r + (int)y) % (int)y);
            else { const T s = (T)((U)r + (U)y); r = (y == (T)-1) ? (T)0 : (T)(s % y); }
          }
          return r;
        }
      }
    }
  });
}

// 128-bit decimal add/sub with overflow -> null (arithmetic.scala:78-125); V_MUL: product known to fit
template <int OP>
__device__ __noinline__ void vm_arith128(const TileInfo ti, const RInstr& ins) {
  vm_loop2<i128, i128>(ti, ins, [](i128 x, i128 y, bool, bool, bool& v) -> i128 {
    if constexpr (OP == V_ADD) { i128 r = (i128)((u128)x + (u128)y); if (((x ^ r) & (y ^ r)) < 0) v = false; return r; }
    else if constexpr (OP == V_SUB) { i128 r = (i128)((u128)x - (u128)y); if (((x ^ y) & (x ^ r)) < 0) v = false; return r; }
    else return (i128)((u128)x * (u128)y);
  });
}

static __device__ __noinline__ void vm_mulw(const TileInfo ti, const RInstr& ins) {
  vm_loop2<int64_t, i128>(ti, ins, [](int64_t x, int64_t y, bool, bool, bool&) -> i128 { return (i128)x * (i128)y; });
}

template <typename T, int OP>
__device__ __noinline__ void vm_compare(const TileInfo ti, const RInstr& ins) {
  vm_loop2<T, int8_t>(ti, ins, [](T x, T y, bool va, bool vb, bool& v) -> int8_t {
    const int c = cmp3<T>(x, y);
    bool r;
    if constexpr (OP == V_EQ) r = c == 0;
    else if constexpr (OP == V_NE) r = c != 0;
    else if constexpr (OP == V_LT) r = c < 0;
    else if constexpr (OP == V_LE) r = c <= 0;
    else if constexpr (OP == V_GT) r = c > 0;
    else if constexpr (OP == V_GE) r = c >= 0;
    else { r = (va && vb) ? (c == 0) : (va == vb); v = true; return (int8_t)r; }  // <=> EqualNullSafe
    return (int8_t)(r && v);
  });
}

// fused conjunct: dst = acc AND (x <cmp> y).  The compiler emits it only when nothing can be NULL, so a WHERE
// chain of n comparisons costs n register passes instead of 2n - 1.
template <typename T>
__device__ __noinline__ void vm_andcmp(const TileInfo ti, const RInstr& ins) {
  const Opnd a = ropnd(ins.a, ti), b = ropnd(ins.b, ti), c = ropnd(ins.c, ti);
  const uint32_t m = (uint32_t)ins.aux;
  char* const dbase = ins.dbase;
  auto f = [m](T x, T y, int8_t acc) -> int8_t { return (int8_t)(acc && ((m >> (cmp3<T>(x, y) + 1)) & 1u)); };
  if (a.stride != 0 && c.stride != 0 && vm_full_tile(ti, ti.tile_rows)) {
    const char* pa = thread_base<T>(a);
    const char* pc = thread_base<int8_t>(c);
    char* pd = dbase + threadIdx.x;
    if (b.stride == 0) {
      const T y = *reinterpret_cast<const T*>(b.base);
      int j0 = 0;
      if constexpr (sizeof(T) <= 8) {
        // column operands come straight from HBM: eight rows per thread in flight before the first use
        for (; j0 + 8 <= ti.K; j0 += 8, pa += 8 * VM_NT * sizeof(T), pc += 8 * VM_NT, pd += 8 * VM_NT) {
          T x[8]; int8_t c[8];
#pragma unroll
          for (int u = 0; u < 8; u++) x[u] = *reinterpret_cast<const T*>(pa + u * VM_NT * sizeof(T));
#pragma unroll
          for (int u = 0; u < 8; u++) c[u] = *reinterpret_cast<const int8_t*>(pc + u * VM_NT);
#pragma unroll
          for (int u = 0; u < 8; u++) pd[u * VM_NT] = f(x[u], y, c[u]);
        }
      }
      for (; j0 + 4 <= ti.K; j0 += 4, pa += 4 * VM_NT * sizeof(T), pc += 4 * VM_NT, pd += 4 * VM_NT) {
        const T x0 = *reinterpret_cast<const T*>(pa), x1 = *reinterpret_cast<const T*>(pa + VM_NT * sizeof(T)),
                x2 = *reinterpret_cast<const T*>(pa + 2 * VM_NT * sizeof(T)), x3 = *reinterpret_cast<const T*>(pa + 3 * VM_NT * sizeof(T));
        const int8_t c0 = *reinterpret_cast<const int8_t*>(pc), c1 = *reinterpret_cast<const int8_t*>(pc + VM_NT),
                     c2 = *reinterpret_cast<const int8_t*>(pc + 2 * VM_NT), c3 = *reinterpret_cast<const int8_t*>(pc + 3 * VM_NT);
        pd[0] = f(x0, y, c0); pd[VM_NT] = f(x1, y, c1); pd[2 * VM_NT] = f(x2, y, c2); pd[3 * VM_NT] = f(x3, y, c3);
      }
      for (; j0 < ti.K; j0++, pa += VM_NT * sizeof(T), pc += VM_NT, pd += VM_NT)
        pd[0] = f(*reinterpret_cast<const T*>(pa), y, *reinterpret_cast<const int8_t*>(pc));
    } else {
      const char* pb = thread_base<T>(b);
      for (int j = 0; j < ti.K; j++, pa += VM_NT * sizeof(T), pb += VM_NT * sizeof(T), pc += VM_NT, pd += VM_NT)
        pd[0] = f(*reinterpret_cast<const T*>(pa), *reinterpret_cast<const T*>(pb), *reinterpret_cast<const int8_t*>(pc));
    }
    return;
  }
  for (int j = 0; j < ti.K; j++) {   // a row is read before it is written and rows are thread private
    VM_ROW_ACTIVE(j, i, g);
    if (act) dbase[i] = f(opnd_ld<T>(a, i), opnd_ld<T>(b, i), opnd_ld<int8_t>(c, i));
  }
}

template <int OP>
__device__ __noinline__ void vm_logic(const TileInfo ti, const RInstr& ins) {
  if constexpr (OP == V_NOT) {
    vm_loop1<int8_t, int8_t>(ti, ins, [](int8_t x, bool& v) -> int8_t { return (int8_t)(v && !x); });
  } else {
    // Kleene logic, predicates.scala:54-153 (NULL_LOGICAL_AND / NULL_LOGICAL_OR)
    vm_loop2<int8_t, int8_t>(ti, ins, [](int8_t xa, int8_t ya, bool va, bool vb, bool& v) -> int8_t {
      const bool x = va && xa, y = vb && ya;
      bool r;
      if constexpr (OP == V_AND) { const bool fa = va && !x, fb = vb && !y; r = x && y; v = (va && vb) || fa || fb; }
      else { r = x || y; v = (va && vb) || x || y; }
      return (int8_t)(r && v);
    });
  }
}

template <typename T>
__device__ __noinline__ void vm_select(const TileInfo ti, const RInstr& ins) {
  typedef typename UnsignedOf<T>::type U;
  switch (ins.op) {
    case V_COALESCE:
      vm_loop2<T, T>(ti, ins, [](T x, T y, bool va, bool vb, bool& v) -> T { v = va || vb; return va ? x : y; });
      break;
    case V_MOV: vm_loop1<T, T>(ti, ins, [](T x, bool&) -> T { return x; }); break;
    case V_NEG:
      vm_loop1<T, T>(ti, ins, [](T x, bool&) -> T { if constexpr (IsFloat<T>::v) return -x; else return (T)((U)0 - (U)x); });
      break;
    case V_ABS:
      vm_loop1<T, T>(ti, ins, [](T x, bool&) -> T {
        if constexpr (IsFloat<T>::v) return (x < 0 || (x == 0 && 1 / (double)x < 0)) ? -x : x;
        else return x < 0 ? (T)((U)0 - (U)x) : x;
      });
      break;
    default: {  // V_IF (conditionalExpressions.scala GpuIf): a NULL predicate takes the else branch
      const Opnd p = ropnd(ins.a, ti), a = ropnd(ins.b, ti), b = ropnd(ins.c, ti);
      const Dst d = rdst(ins, sizeof(T));
          for (int j = 0; j < ti.K; j++) {
        VM_ROW_ACTIVE(j, i, g);
        if (!act) continue;
        const bool t = opnd_valid(p, i, g) && opnd_ld<int8_t>(p, i);
        const T r = t ? opnd_ld<T>(a, i) : opnd_ld<T>(b, i);
        const bool v = t ? opnd_valid(a, i, g) : opnd_valid(b, i, g);
        dst_st<T>(d, i, r, v);
      }
    } break;
  }
}

// correctly rounded signed 128-bit -> double (keep 64 significant bits + sticky, then scale)
__device__ __forceinline__ double i128_to_double(i128 x) {
  bool neg = x < 0;
  u128 m = neg ? (u128)0 - (u128)x : (u128)x;
  uint64_t hi = (uint64_t)(m >> 64), lo = (uint64_t)m;
  double r;
  if (hi == 0) r = (double)lo;
  else {
    int lz = __clzll((long long)hi);
    int sh = 64 - lz;  // bits shifted out of the low word
    uint64_t top = (uint64_t)(m >> sh);
    bool sticky = (m & ((((u128)1) << sh) - 1)) != 0;
    top |= sticky ? 1ull : 0ull;
    r = ldexp((double)top, sh);
  }
  return neg ? -r : r;
}
template <typename S, typename D> struct CastVia { __device__ static __forceinline__ D f(S x) { return (D)x; } };
template <> struct CastVia<i128, double> { __device__ static __forceinline__ double f(i128 x) { return i128_to_double(x); } };
template <> struct CastVia<i128, float> { __device__ static __forceinline__ float f(i128 x) { return (float)i128_to_double(x); } };

// GpuCast.scala:295 doCast, numeric subset.  Integral narrowing wraps (Java semantics); float ->
// integral follows Java (NaN -> 0, saturating) via int/long then narrows.
template <typename S, typename D>
__device__ __forceinline__ D cast_val(S x) {
  if constexpr (IsFloat<S>::v && !IsFloat<D>::v) {
    if constexpr (sizeof(D) >= 8) {
      if (x != x) return (D)0;
      if (x >= (S)9223372036854775807.0) return (D)0x7fffffffffffffffLL;
      if (x <= (S)-9223372036854775808.0) return (D)(-0x7fffffffffffffffLL - 1);
      return (D)(long long)x;
    } else {
      int v;
      if (x != x) v = 0;
      else if (x >= (S)2147483647.0) v = 0x7fffffff;
      else if (x <= (S)-2147483648.0) v = -0x7fffffff - 1;
      else v = (int)x;
      return (D)v;
    }
  } else {
    return CastVia<S, D>::f(x);
  }
}
template <typename S, typename D>
__device__ __noinline__ void vm_cast2(const TileInfo ti, const RInstr& ins) {
  vm_loop1<S, D>(ti, ins, [](S x, bool&) -> D { return cast_val<S, D>(x); });
}
template <typename S>
__device__ __forceinline__ void vm_cast1(const TileInfo ti, const RInstr& ins) {
  switch (ins.mt2) {
    case MT_I8: vm_cast2<S, int8_t>(ti, ins); break;
    case MT_I16: vm_cast2<S, int16_t>(ti, ins); break;
    case MT_I32: vm_cast2<S, int32_t>(ti, ins); break;
    case MT_I64: vm_cast2<S, int64_t>(ti, ins); break;
    case MT_I128: vm_cast2<S, i128>(ti, ins); break;
    case MT_F32: vm_cast2<S, float>(ti, ins); break;
    default: vm_cast2<S, double>(ti, ins); break;
  }
}

// divide a 256-bit magnitude (4 x u64 little endian) by a u64, returning the remainder
__device__ __forceinline__ uint64_t div256_u64(uint64_t q[4], uint64_t dv) {
  u128 rem = 0;
  for (int k = 3; k >= 0; k--) {
    u128 cur = (rem << 64) | q[k];
    q[k] = (uint64_t)(cur / dv);
    rem = cur % dv;
  }
  return (uint64_t)rem;
}

template <typename T>
__device__ __noinline__ void vm_decimal(const TileInfo ti, const RInstr& ins) {
  const i128 p = pow10_i128(ins.aux);
  if (ins.op == V_RESCALE_UP) {
    const i128 maxv = (i128)((((u128)1) << (8 * sizeof(T) - 1)) - 1);
    const i128 lim = maxv / p;
    vm_loop1<T, T>(ti, ins, [p, lim](T xx, bool& v) -> T {
      const i128 x = (i128)xx;
      if (x > lim || x < -lim) v = false;  // |x| * 10^aux does not fit T
      return (T)(i128)((u128)x * (u128)p);
    });
  } else if (ins.op == V_RESCALE_DOWN) {  // HALF_UP (away from zero), as BigDecimal.setScale
    vm_loop1<T, T>(ti, ins, [p](T xx, bool&) -> T {
      const i128 x = (i128)xx;
      const bool neg = x < 0;
      const u128 m = neg ? (u128)0 - (u128)x : (u128)x;
      u128 q = m / (u128)p;
      const u128 r = m % (u128)p;
      if (r * 2 >= (u128)p) q += 1;
      return (T)(neg ? -(i128)q : (i128)q);
    });
  } else {  // V_CHECK_PREC
    vm_loop1<T, T>(ti, ins, [p](T x, bool& v) -> T { const i128 xx = (i128)x; if (xx >= p || xx <= -p) v = false; return x; });
  }
}

// DecimalUtils.multiply128 (arithmetic.scala:470-512 longMultiply): exact 256-bit product,
// HALF_UP to the result scale, NULL when the result needs more than 38 digits.
template <typename TB>
static __device__ __noinline__ void vm_muldec(const TileInfo ti, const RInstr& ins) {
  const int k = ins.aux;
  const u128 p38 = (u128)pow10_i128(38);
  vm_loop2x<i128, i128, TB>(ti, ins, [k, p38](i128 x, TB yy, bool, bool, bool& v) -> i128 {
    const i128 y = (i128)yy;
    const bool neg = (x < 0) != (y < 0);
    const u128 mx = x < 0 ? (u128)0 - (u128)x : (u128)x, my = y < 0 ? (u128)0 - (u128)y : (u128)y;
    const uint64_t x0 = (uint64_t)mx, x1 = (uint64_t)(mx >> 64), y0 = (uint64_t)my, y1 = (uint64_t)(my >> 64);
    uint64_t q[4];
    const u128 p00 = (u128)x0 * y0, p01 = (u128)x0 * y1, p10 = (u128)x1 * y0, p11 = (u128)x1 * y1;
    q[0] = (uint64_t)p00;
    const u128 mid = (p00 >> 64) + (uint64_t)p01 + (uint64_t)p10;
    q[1] = (uint64_t)mid;
    const u128 hi = (mid >> 64) + (p01 >> 64) + (p10 >> 64) + (uint64_t)p11;
    q[2] = (uint64_t)hi;
    q[3] = (uint64_t)((hi >> 64) + (p11 >> 64));
    if (k > 0) {
      // divide by 10^k (k <= 39) in u64 steps of at most 19 digits.  Only the last step's remainder r decides HALF_UP:
      // the whole remainder is r * L + low with low < L (L = product of the earlier divisors), and that last divisor
      // d = 10^j is even, so  r * L + low >= (d / 2) * L  exactly when  r >= d / 2.
      uint64_t d = 1, r = 0;
      for (int left = k; left > 0;) {
        const int j = left > 19 ? 19 : left;
        d = 1; for (int t = 0; t < j; t++) d *= 10ull;
        r = div256_u64(q, d);
        left -= j;
      }
      if (r >= d / 2) { for (int t = 0; t < 4; t++) { if (++q[t] != 0) break; } }
    }
    const u128 mag = ((u128)q[1] << 64) | q[0];
    if (q[2] || q[3] || mag >= p38) v = false;
    return neg ? -(i128)mag : (i128)mag;
  });
}

// Decimal divide (arithmetic.scala:903-1000 GpuDecimalDivideBase.longDivide -> DecimalUtils.divide128):
// exact 256-bit numerator |a| * 10^k, restoring long division by |b|, HALF_UP, NULL on zero divisor
// or when the quotient needs more than 38 digits.
static __device__ __noinline__ void vm_divdec(const TileInfo ti, const RInstr& ins) {
  const int k = ins.aux;
  const u128 p38 = (u128)pow10_i128(38);
  const u128 pk = (u128)pow10_i128(k);
  vm_loop2<i128, i128>(ti, ins, [pk, p38](i128 x, i128 y, bool, bool, bool& v) -> i128 {
    if (y == 0) { v = false; return (i128)0; }
    const bool neg = (x < 0) != (y < 0);
    const u128 mx = x < 0 ? (u128)0 - (u128)x : (u128)x, my = y < 0 ? (u128)0 - (u128)y : (u128)y;
    // 256-bit numerator = mx * pk
    const uint64_t x0 = (uint64_t)mx, x1 = (uint64_t)(mx >> 64), y0 = (uint64_t)pk, y1 = (uint64_t)(pk >> 64);
    const u128 p00 = (u128)x0 * y0, p01 = (u128)x0 * y1, p10 = (u128)x1 * y0, p11 = (u128)x1 * y1;
    const u128 mid = (p00 >> 64) + (uint64_t)p01 + (uint64_t)p10;
    const u128 lo = ((u128)(uint64_t)mid << 64) | (uint64_t)p00;
    const u128 hi = (mid >> 64) + (p01 >> 64) + (p10 >> 64) + p11;
    if (hi >= my) { v = false; return (i128)0; }  // quotient would not fit 128 bits
    u128 rem = hi, q = 0;
    for (int i = 127; i >= 0; i--) {
      const bool top = (rem >> 127) != 0;
      rem = (rem << 1) | ((lo >> i) & 1);
      if (top || rem >= my) { rem -= my; q |= (u128)1 << i; }
    }
    if (rem >= my - rem) q += 1;  // 2*rem >= my, HALF_UP
    if (q >= p38) { v = false; return (i128)0; }
    return neg ? -(i128)q : (i128)q;
  });
}

// the doubles nearest to 10^0 .. 10^38 (multiplying 10.0s together lands 1 ulp low for 10^25..27, 10^30..32, 10^36..38)
static __device__ const double kPow10F64[39] = {
    1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19,
    1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27, 1e28, 1e29, 1e30, 1e31, 1e32, 1e33, 1e34, 1e35, 1e36, 1e37, 1e38};

// one correctly rounded integer -> double, then one IEEE division by the correctly rounded 10^scale
template <typename T>
__device__ __noinline__ void vm_dec2f64(const TileInfo ti, const RInstr& ins) {
  const double dv = kPow10F64[ins.aux];
  vm_loop1<T, double>(ti, ins, [dv](T x, bool&) -> double { return CastVia<T, double>::f(x) / dv; });
}

template <typename T>
__device__ __noinline__ void vm_normnz(const TileInfo ti, const RInstr& ins) {
  vm_loop1<T, T>(ti, ins, [](T x, bool&) -> T {  // NormalizeFloatingNumbers.scala:29-38: canonical NaN, -0.0 -> 0.0
    if (x != x) return (T)__longlong_as_double(0x7ff8000000000000LL);
    if (x == (T)0) return (T)0;
    return x;
  });
}

static __device__ __noinline__ void vm_year(const TileInfo ti, const RInstr& ins) {
  vm_loop1<int32_t, int32_t>(ti, ins, [](int32_t days, bool&) -> int32_t {  // proleptic Gregorian civil-from-days
    const int z = days + 719468;
    const int era = (z >= 0 ? z : z - 146096) / 146097;
    const unsigned doe = (unsigned)(z - era * 146097);
    const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int y = (int)yoe + era * 400;
    const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const unsigned mp = (5 * doy + 2) / 153;
    const int m = mp < 10 ? mp + 3 : mp - 9;
    return y + (m <= 2);
  });
}

static __device__ __noinline__ void vm_isnull(const TileInfo ti, const RInstr& ins) {
  const Opnd a = ropnd(ins.a, ti);
  const Dst d = rdst(ins, 1);
  const bool want_null = ins.op == V_ISNULL;
  for (int j = 0; j < ti.K; j++) { VM_ROW_ACTIVE(j, i, g); if (act) dst_st<int8_t>(d, i, (int8_t)(opnd_valid(a, i, g) != want_null), true); }
}


// ---- string predicates -------------------------------------------------------------------------------------------
// Strings never enter the register file: a predicate reads (offsets, chars) of its column operand straight from
// global memory and leaves a BOOL8 register.  Literals sit in the program's pool (shared memory).
__device__ __forceinline__ int utf8_len(uint8_t lead) { return lead < 0x80 ? 1 : ((lead >> 5) == 6 ? 2 : ((lead >> 4) == 14 ? 3 : ((lead >> 3) == 30 ? 4 : 1))); }
// UTF8String.substringSQL(pos, len) as the reference restates it (stringFunctions.scala:540-600): code-point based,
// start = pos < 0 ? pos + nchars : (pos > 0 ? pos - 1 : 0), end = clamp(start + len, 0, INT_MAX), start < 0 -> 0
__device__ __forceinline__ void str_window(const uint8_t*& p, int& n, int64_t pos, int64_t len) {
  int nchars = 0;
  for (int k = 0; k < n; k++) nchars += (p[k] & 0xc0) != 0x80;
  int64_t start = pos < 0 ? pos + nchars : (pos > 0 ? pos - 1 : 0);
  int64_t end = start + len;
  if (end < 0) end = 0;
  if (end > 0x7fffffffLL) end = 0x7fffffffLL;
  if (start < 0) start = 0;
  if (start >= end || start >= nchars) { n = 0; return; }
  int b0 = 0, c = 0;
  while (b0 < n && c < start) { b0 += utf8_len(p[b0]); c++; }
  int b1 = b0;
  while (b1 < n && c < end) { b1 += utf8_len(p[b1]); c++; }
  if (b1 > n) b1 = n;
  p += b0; n = b1 - b0;
}
__device__ __forceinline__ int str_cmp(const uint8_t* a, int an, const uint8_t* b, int bn) {
  const int m = an < bn ? an : bn;
  for (int k = 0; k < m; k++) { const int d = (int)a[k] - (int)b[k]; if (d) return d; }
  return an - bn;
}
__device__ __forceinline__ bool str_like(const uint8_t* s, int sn, const uint8_t* p, int pn, uint8_t esc) {
  int si = 0, pi = 0, star_p = -1, star_s = 0;
  while (si < sn) {
    bool ok = false;
    if (pi < pn) {
      const uint8_t c = p[pi];
      if (c == esc && pi + 1 < pn) { if (s[si] == p[pi + 1]) { si++; pi += 2; ok = true; } }
      else if (c == '%') { star_p = ++pi; star_s = si; ok = true; }
      else if (c == '_') { si += utf8_len(s[si]); pi++; ok = true; }
      else if (c == s[si]) { si++; pi++; ok = true; }
    }
    if (ok) continue;
    if (star_p < 0) return false;
    pi = star_p; star_s += utf8_len(s[star_s]); si = star_s;
  }
  while (pi < pn && p[pi] == '%') pi++;
  return pi == pn;
}
__device__ __forceinline__ bool str_pred(int kind, const uint8_t* a, int an, const uint8_t* b, int bn, uint8_t esc) {
  switch (kind) {
    case SP_EQ: return an == bn && str_cmp(a, an, b, bn) == 0;
    case SP_NE: return !(an == bn && str_cmp(a, an, b, bn) == 0);
    case SP_LT: return str_cmp(a, an, b, bn) < 0;
    case SP_LE: return str_cmp(a, an, b, bn) <= 0;
    case SP_GT: return str_cmp(a, an, b, bn) > 0;
    case SP_GE: return str_cmp(a, an, b, bn) >= 0;
    case SP_STARTS: return bn <= an && str_cmp(a, bn, b, bn) == 0;
    case SP_ENDS: return bn <= an && str_cmp(a + (an - bn), bn, b, bn) == 0;
    case SP_CONTAINS: {
      if (bn == 0) return true;
      for (int k = 0; k + bn <= an; k++) if (a[k] == b[0] && str_cmp(a + k, bn, b, bn) == 0) return true;
      return false;
    }
    default: return str_like(a, an, b, bn, esc);
  }
}
__device__ __forceinline__ const int32_t* ropnd_offsets(const ROpnd& o) {  // string column operand: the offsets pointer rides in (stride, tile_step)
  const int32_t* p; memcpy(&p, &o.stride, sizeof(p)); return p;
}
static __device__ __noinline__ void vm_strpred(const TileInfo ti, const RInstr& ins) {
  const uint8_t* achars = reinterpret_cast<const uint8_t*>(ins.a.base);
  const int32_t* aoff = ropnd_offsets(ins.a);
  const uint32_t* avalid = reinterpret_cast<const uint32_t*>(ins.a.vptr);
  const bool b_lit = ins.mt2 == 1;
  const uint8_t* bchars = reinterpret_cast<const uint8_t*>(ins.b.base);
  const int32_t* boff = b_lit ? nullptr : ropnd_offsets(ins.b);
  const uint32_t* bvalid = reinterpret_cast<const uint32_t*>(ins.b.vptr);
  const int blit_len = b_lit ? ins.b.stride : 0;
  const bool window = ins.c.base != nullptr;
  int64_t wpos = 0, wlen = 0;
  if (window) { wpos = reinterpret_cast<const int64_t*>(ins.c.base)[0]; wlen = reinterpret_cast<const int64_t*>(ins.c.base)[1]; }
  const int kind = ins.aux & 0xff;
  const uint8_t esc = (uint8_t)((ins.aux >> 8) & 0xff);
  const Dst d = rdst(ins, 1);
  for (int j = 0; j < ti.K; j++) {
    VM_ROW_ACTIVE(j, i, g);
    if (!act) continue;
    bool v = (ins.a.vkind == 0 || (ins.a.vkind == 2 && bit_get(avalid, g))) && ins.b.vkind != 3;
    if (!b_lit) v = v && (ins.b.vkind == 0 || (ins.b.vkind == 2 && bit_get(bvalid, g)));
    bool r = false;
    if (v) {
      const int32_t a0 = aoff[g];
      const uint8_t* ap = achars + a0; int an = aoff[g + 1] - a0;
      if (window) str_window(ap, an, wpos, wlen);
      const uint8_t* bp = bchars; int bn = blit_len;
      if (!b_lit) { const int32_t b0 = boff[g]; bp = bchars + b0; bn = boff[g + 1] - b0; }
      r = str_pred(kind, ap, an, bp, bn, esc);
    }
    dst_st<int8_t>(d, i, (int8_t)(r && v), v);
  }
}

#define VM_TYPES_INT_FLOAT(fn, ...)                         \
  switch (ins.mt) {                                         \
    case MT_I8: fn<int8_t, ##__VA_ARGS__>(ti, ins); break;  \
    case MT_I16: fn<int16_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_I32: fn<int32_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_I64: fn<int64_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_F32: fn<float, ##__VA_ARGS__>(ti, ins); break;  \
    case MT_F64: fn<double, ##__VA_ARGS__>(ti, ins); break; \
    default: break;                                         \
  }
#define VM_TYPES_ALL(fn, ...)                               \
  switch (ins.mt) {                                         \
    case MT_I8: fn<int8_t, ##__VA_ARGS__>(ti, ins); break;  \
    case MT_I16: fn<int16_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_I32: fn<int32_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_I64: fn<int64_t, ##__VA_ARGS__>(ti, ins); break;\
    case MT_I128: fn<i128, ##__VA_ARGS__>(ti, ins); break;  \
    case MT_F32: fn<float, ##__VA_ARGS__>(ti, ins); break;  \
    default: fn<double, ##__VA_ARGS__>(ti, ins); break;     \
  }
#define VM_ARITH_CASE(OP)                                                                       \
  case OP: if (ins.mt == MT_I128) vm_arith128<OP>(ti, ins); else { VM_TYPES_INT_FLOAT(vm_arith, OP) } break;
#define VM_CMP_CASE(OP) case OP: VM_TYPES_ALL(vm_compare, OP) break;

// Execute instructions [first, last) over this CTA's tile.  No barrier is needed: registers are thread private.
static __device__ __noinline__ void vm_run(const TileInfo ti, const RInstr* __restrict__ code, int first, int last) {
  for (int pc = first; pc < last; pc++) {
    const RInstr& ins = code[pc];
    switch (ins.op) {
      VM_ARITH_CASE(V_ADD) VM_ARITH_CASE(V_SUB) VM_ARITH_CASE(V_MUL)
      case V_DIV: VM_TYPES_INT_FLOAT(vm_arith, V_DIV) break;
      case V_MOD: VM_TYPES_INT_FLOAT(vm_arith, V_MOD) break;
      case V_PMOD: VM_TYPES_INT_FLOAT(vm_arith, V_PMOD) break;
      VM_CMP_CASE(V_EQ) VM_CMP_CASE(V_NE) VM_CMP_CASE(V_LT) VM_CMP_CASE(V_LE) VM_CMP_CASE(V_GT) VM_CMP_CASE(V_GE) VM_CMP_CASE(V_EQNS)
      case V_AND: vm_logic<V_AND>(ti, ins); break;
      case V_OR: vm_logic<V_OR>(ti, ins); break;
      case V_NOT: vm_logic<V_NOT>(ti, ins); break;
      case V_ISNULL: case V_ISNOTNULL: vm_isnull(ti, ins); break;
      case V_COALESCE: case V_IF: case V_MOV: case V_NEG: case V_ABS:
        VM_TYPES_ALL(vm_select)
        break;
      case V_CAST: VM_TYPES_ALL(vm_cast1) break;
      case V_RESCALE_UP: case V_RESCALE_DOWN: case V_CHECK_PREC:
        switch (ins.mt) {
          case MT_I32: vm_decimal<int32_t>(ti, ins); break;
          case MT_I64: vm_decimal<int64_t>(ti, ins); break;
          default: vm_decimal<i128>(ti, ins); break;
        }
        break;
      case V_MULW: vm_mulw(ti, ins); break;
      case V_MULDEC: if (ins.mt2 == MT_I64) vm_muldec<int64_t>(ti, ins); else vm_muldec<i128>(ti, ins); break;
      case V_DIVDEC: vm_divdec(ti, ins); break;
      case V_DEC2F64:
        switch (ins.mt) {
          case MT_I32: vm_dec2f64<int32_t>(ti, ins); break;
          case MT_I64: vm_dec2f64<int64_t>(ti, ins); break;
          default: vm_dec2f64<i128>(ti, ins); break;
        }
        break;
      case V_NORM_NAN_ZERO: if (ins.mt == MT_F32) vm_normnz<float>(ti, ins); else vm_normnz<double>(ti, ins); break;
      case V_YEAR: vm_year(ti, ins); break;
      case V_ANDCMP: VM_TYPES_ALL(vm_andcmp) break;
      case V_STRPRED: vm_strpred(ti, ins); break;
      default: break;
    }
  }
}

// context for one tile
__device__ __forceinline__ VMCtx vm_ctx(const VMProgramHeader* hdr, const VMInputs* in, char* smem, int64_t tile, int64_t nrows) {
  VMCtx cx;
  cx.hdr = hdr; cx.in = in; cx.smem = smem; cx.tile_rows = hdr->tile_rows; cx.K = hdr->tile_rows / VM_NT;
  cx.tile_base = tile * (int64_t)hdr->tile_rows; cx.nrows = nrows; cx.rowmask = 0xffffffffu; cx.stage_off = 0;
  return cx;
}

// Input columns staged in shared memory by TMA bulk copies (cp.async.bulk + mbarrier, double buffered): the row loops of
// the VM then touch shared memory only, and the HBM stream of tile k+1 overlaps the evaluation of tile k.
constexpr int VM_MAX_STAGED = 24;
struct VMStage {
  int32_t n;                           // staged columns (0 = staging off)
  int32_t tile_rows;                   // rows per tile of the staged kernel (overrides the program's own geometry)
  int32_t buf_bytes;                   // bytes of ONE stage buffer (all staged columns of a tile)
  int32_t pad;
  int8_t slot_of_col[VM_MAX_COLS];     // table column -> staged slot, -1 = read from global
  int32_t width[VM_MAX_STAGED];
  int32_t off[VM_MAX_STAGED];          // byte offset of the column inside a stage buffer
  const char* src[VM_MAX_STAGED];
};

// ---- TMA 1-D bulk copy + mbarrier (PTX; SASS: UBLKCP + SYNCS) -------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "B2_MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra B2_MBAR_DONE;\n"
      "bra B2_MBAR_WAIT;\n"
      "B2_MBAR_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completes on `bar`
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one thread: start the copies of every staged column of tile `tile` into stage buffer `buf`
__device__ __forceinline__ void vm_stage_issue(const VMStage& st, char* stage_base, int buf, int64_t tile, int64_t nrows, uint64_t* bar) {
  const int64_t row0 = tile * (int64_t)st.tile_rows;
  const int64_t rows = min((int64_t)st.tile_rows, nrows - row0);
  uint32_t total = 0;
  for (int k = 0; k < st.n; k++) total += (uint32_t)((rows * st.width[k] + 15) & ~15LL);
  fence_proxy_async();    // the buffer was read through the generic proxy by the previous tile
  mbar_expect_tx(bar, total);
  for (int k = 0; k < st.n; k++) {
    const uint32_t bytes = (uint32_t)((rows * st.width[k] + 15) & ~15LL);   // column buffers are padded to 64 B
    tma_bulk_g2s(stage_base + (size_t)buf * st.buf_bytes + st.off[k], st.src[k] + row0 * st.width[k], bytes, bar);
  }
}
#endif

constexpr int VM_SMEM_CODE = 64;  // instructions per program (resolved form lives in shared memory)
struct VMShared {
  VMProgramHeader hdr;
  RInstr code[VM_SMEM_CODE];
};
// cooperative load: header into shared memory, then one thread per instruction resolves its operands
static __device__ __forceinline__ const RInstr* vm_load_program(VMShared& sh, const VMProgramHeader* g_hdr, const VMInstr* g_code,
                                                                 const VMInputs& in, char* regs, const VMStage* stage = nullptr,
                                                                 char* stage_base = nullptr, int fixed_tile_rows = 0) {
  const int* src = reinterpret_cast<const int*>(g_hdr);
  int* dst = reinterpret_cast<int*>(&sh.hdr);
  for (int k = threadIdx.x; k < (int)(sizeof(VMProgramHeader) / 4); k += blockDim.x) dst[k] = src[k];
  __syncthreads();
  // the staged kernel picks its own tile size (registers + two stage buffers per tile); a kernel whose tile is fixed by
  // something else (the radix group-by's fused first pass) passes it as fixed_tile_rows (a multiple of VM_NT, <= 4096)
  const int own_rows = (stage && stage->n > 0) ? stage->tile_rows : fixed_tile_rows;
  if (own_rows > 0) {
    if (threadIdx.x == 0) { sh.hdr.tile_rows = own_rows; sh.hdr.smem_bytes = sh.hdr.bytes_per_row * own_rows; }
    __syncthreads();
  }
  const int n = sh.hdr.ninstr;
  const int tile_rows = sh.hdr.tile_rows;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const VMInstr& g = g_code[k];
    RInstr r;
    r.op = g.op; r.mt = g.mt; r.mt2 = g.mt2; r.dst_nullable = g.dst_nullable; r.aux = g.aux; r.pad = 0;
    r.dbase = regs + (size_t)sh.hdr.regs[g.dst].off * tile_rows;
    r.dvb = reinterpret_cast<uint8_t*>(regs + (size_t)sh.hdr.regs[g.dst].voff * tile_rows);
    const VMOperand* ops[3] = {&g.a, &g.b, &g.c};
    ROpnd* outs[3] = {&r.a, &r.b, &r.c};
    // operand width = the instruction's input machine type, except boolean operands of logic ops / IF predicate
    for (int j = 0; j < 3; j++) {
      const VMOperand& o = *ops[j];
      ROpnd q; q.pad = 0; q.vptr = nullptr; q.tile_step = 0;
      int width = mt_width(g.mt);
      if (g.op == V_AND || g.op == V_OR || g.op == V_NOT || (g.op == V_IF && j == 0)) width = 1;
      if (g.op == V_MULDEC && j == 1) width = mt_width(g.mt2);
      if (g.op == V_ANDCMP && j == 2) width = 1;   // the accumulated predicate
      if (g.op == V_STRPRED) {   // string operands: see vm_strpred
        q.base = nullptr; q.stride = 0; q.vkind = 0;
        if (j == 2) { if (o.kind == OK_LIT) q.base = reinterpret_cast<const char*>(&o.lo); }
        else if (o.kind == OK_COL) {
          q.base = reinterpret_cast<const char*>(in.data[o.idx]); q.vptr = in.valid[o.idx];
          q.vkind = (o.nullable && in.valid[o.idx]) ? 2 : 0;
          const int32_t* offs = in.offsets[o.idx]; memcpy(&q.stride, &offs, sizeof(offs));
        } else if (o.kind == OK_LIT) {
          q.base = sh.hdr.lits + o.lo; q.stride = (int32_t)o.hi; q.vkind = o.lit_null ? 3 : 0;
        }
        *outs[j] = q;
        continue;
      }
      if (o.kind == OK_REG) {
        q.base = regs + (size_t)sh.hdr.regs[o.idx].off * tile_rows; q.stride = width;
        q.vkind = o.nullable ? 1 : 0; q.vptr = regs + (size_t)sh.hdr.regs[o.idx].voff * tile_rows;
      } else if (o.kind == OK_COL) {
        q.base = reinterpret_cast<const char*>(in.data[o.idx]); q.stride = width; q.tile_step = width;
        q.vptr = in.valid[o.idx]; q.vkind = (o.nullable && in.valid[o.idx]) ? 2 : 0;
        if (stage && stage->n > 0 && stage->slot_of_col[o.idx] >= 0) {   // this column's tile sits in shared memory
          q.base = stage_base + stage->off[stage->slot_of_col[o.idx]]; q.tile_step = 0; q.pad = 1;
        }
      } else {
        q.base = reinterpret_cast<const char*>(&o.lo); q.stride = 0; q.vkind = o.lit_null ? 3 : 0;
      }
      *outs[j] = q;
    }
    sh.code[k] = r;
  }
  __syncthreads();
  return sh.code;
}

#endif  // __CUDACC__

// host-side compiled program
struct Program {
  VMProgramHeader hdr;
  std::vector<VMInstr> code;
  std::vector<int> col_dtype;          // expected dtype of each referenced input column (-1 unused)
  std::vector<int> out_dtype, out_scale, out_precision;
  std::vector<uint8_t> out_nullable;
  DevBuf d_hdr, d_code;                // device copies
};
Program* program_from(b2_handle h);
void set_tile_geometry(VMProgramHeader& hdr, int bytes_per_row);

}  // namespace b2
