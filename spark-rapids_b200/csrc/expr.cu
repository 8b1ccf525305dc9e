// expr.cu — host side of a1: bound expression trees with Spark types and their compilation into a
// VM program (vm.cuh).  Mirrors what GpuExpression.convertToAst + ast.CompiledExpression do in
// the reference (GpuExpressions.scala:197; basicPhysicalOperators.scala:865-884), including the
// Spark decimal result-type rules the reference applies in arithmetic.scala:411-640
// (DecimalMultiplyChecks) and Spark's DecimalPrecision.
#include <algorithm>
#include <map>
#include "vm.cuh"

namespace b2 {

struct Expr {
  std::atomic<int> refs{1};
  int op = 0;            // 0 = column, -1 = literal, -2 = cast, else b2_expr_op
  int dtype = B2_INT64, precision = 0, scale = 0;
  bool nullable = false;
  int column = -1;
  int64_t lit_lo = 0, lit_hi = 0;
  bool lit_null = false;
  std::string str;       // STRING literal bytes (UTF-8)
  int escape = '\\';     // LIKE escape character
  std::vector<Expr*> kids;
  ~Expr() {
    for (auto* k : kids)
      if (k->refs.fetch_sub(1) == 1) delete k;
  }
};
static Expr* expr_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null expression handle");
  return reinterpret_cast<Expr*>((intptr_t)h);
}
Program* program_from(b2_handle h) {
  if (!h) throw Error(B2_ERR_INVALID, "null program handle");
  return reinterpret_cast<Program*>((intptr_t)h);
}

static int mt_of(int dtype) {
  switch (dtype) {
    case B2_BOOL8: case B2_INT8: return MT_I8;
    case B2_INT16: return MT_I16;
    case B2_INT32: case B2_DATE32: case B2_DECIMAL32: return MT_I32;
    case B2_INT64: case B2_TIMESTAMP_US: case B2_DECIMAL64: return MT_I64;
    case B2_DECIMAL128: return MT_I128;
    case B2_FLOAT32: return MT_F32;
    case B2_FLOAT64: return MT_F64;
  }
  throw Error(B2_ERR_UNSUPPORTED, "expression over dtype " + std::to_string(dtype) + " is not supported");
}
static int decimal_dtype_for(int precision) {  // DecimalUtil.scala:24-40
  return precision <= 9 ? B2_DECIMAL32 : (precision <= 18 ? B2_DECIMAL64 : B2_DECIMAL128);
}
static int default_precision(int dtype) {
  switch (dtype) {  // Spark DecimalType.forType
    case B2_INT8: return 3; case B2_INT16: return 5; case B2_INT32: return 10; case B2_INT64: return 20;
  }
  return 0;
}
// DecimalType.adjustPrecisionScale (allowPrecisionLoss = true)
static void adjust_precision_scale(int& p, int& s) {
  if (p <= 38) return;
  int int_digits = p - s;
  int min_scale = std::min(s, 6);
  int adj = std::max(38 - int_digits, min_scale);
  p = 38; s = adj;
}

// ------------------------------------------------------------------------------------------------
struct Val {  // a compiled sub-expression
  VMOperand o;
  int mt;
  int dtype, precision, scale;
  bool nullable;
  bool win = false;          // STRING column seen through Substring(pos, len): only a string predicate can consume it
  int64_t wpos = 0, wlen = 0;
};

struct Compiler {
  Program* prog;
  struct Slot { int off; int width; };
  std::map<int, std::vector<int>> free_slots;  // width -> free offsets
  int bump = 0;
  std::vector<int> reg_width;
  std::vector<bool> reg_pinned;

  int alloc_slot(int width) {
    auto& fl = free_slots[width];
    if (!fl.empty()) { int o = fl.back(); fl.pop_back(); return o; }
    // offsets are in bytes PER ROW; the kernel scales them by the tile's row count (a multiple of
    // 256), so every slot base stays 256-byte aligned
    int o = bump; bump += width;
    return o;
  }
  int alloc_reg(int mt, bool nullable) {
    int r = (int)reg_width.size();
    if (r >= VM_MAX_REGS) throw Error(B2_ERR_UNSUPPORTED, "expression needs too many registers");
    int w = mt_width(mt);
    reg_width.push_back(w);
    reg_pinned.push_back(false);
    prog->hdr.regs[r].off = alloc_slot(w);
    prog->hdr.regs[r].voff = nullable ? alloc_slot(1) : 0;
    reg_nullable.push_back(nullable);
    return r;
  }
  std::vector<bool> reg_nullable;
  void release(const Val& v) {
    if (v.o.kind != OK_REG) return;
    int r = v.o.idx;
    if (reg_pinned[r]) return;
    free_slots[reg_width[r]].push_back(prog->hdr.regs[r].off);
    if (reg_nullable[r]) free_slots[1].push_back(prog->hdr.regs[r].voff);
    reg_pinned[r] = true;  // never release twice
  }

  static VMOperand none() { VMOperand o; memset(&o, 0, sizeof(o)); return o; }
  static VMOperand lit(int64_t lo, int64_t hi, bool is_null) {
    VMOperand o = none(); o.kind = OK_LIT; o.lo = lo; o.hi = hi; o.lit_null = is_null; o.nullable = is_null; return o;
  }

  Val emit(int op, int mt, int mt2, int out_mt, bool out_nullable, int aux, const Val* a, const Val* b, const Val* c,
           int dtype, int precision, int scale) {
    for (const Val* v : {a, b, c})
      if (v && v->dtype == B2_STRING && !((op == V_ISNULL || op == V_ISNOTNULL) && v->o.kind == OK_COL && !v->win))
        throw Error(B2_ERR_UNSUPPORTED, "string-valued expressions (only string predicates and IS [NOT] NULL are compiled)");
    VMInstr ins; memset(&ins, 0, sizeof(ins));
    ins.op = (uint8_t)op; ins.mt = (uint8_t)mt; ins.mt2 = (uint8_t)mt2; ins.aux = aux;
    ins.a = a ? a->o : none(); ins.b = b ? b->o : none(); ins.c = c ? c->o : none();
    // sources may be recycled for the destination: every handler reads a row before writing it
    if (a) release(*a);
    if (b) release(*b);
    if (c) release(*c);
    int r = alloc_reg(out_mt, out_nullable);
    ins.dst = r; ins.dst_nullable = out_nullable;
    prog->code.push_back(ins);
    Val v; v.o = none(); v.o.kind = OK_REG; v.o.idx = r; v.o.nullable = out_nullable;
    v.mt = out_mt; v.dtype = dtype; v.precision = precision; v.scale = scale; v.nullable = out_nullable;
    return v;
  }

  int lit_used = 0;
  int64_t intern(const std::string& bytes) {   // string literal -> offset in the program's pool
    if (lit_used + (int)bytes.size() > VM_LIT_BYTES) throw Error(B2_ERR_UNSUPPORTED, "string literals of one program exceed 512 bytes");
    const int off = lit_used;
    memcpy(prog->hdr.lits + off, bytes.data(), bytes.size());
    lit_used += (int)bytes.size();
    return off;
  }
  Val emit_strpred(int kind, const Val& a, const Val& b, int escape) {
    if (a.o.kind != OK_COL) throw Error(B2_ERR_UNSUPPORTED, "string predicate: the left side must be a STRING column");
    if (b.o.kind != OK_COL && b.o.kind != OK_LIT) throw Error(B2_ERR_UNSUPPORTED, "string predicate: the right side must be a column or a literal");
    if (b.win) throw Error(B2_ERR_UNSUPPORTED, "Substring on the right side of a string predicate");
    VMInstr ins; memset(&ins, 0, sizeof(ins));
    ins.op = V_STRPRED; ins.mt = MT_I8; ins.mt2 = b.o.kind == OK_LIT ? 1 : 0; ins.aux = kind | ((escape & 0xff) << 8);
    ins.a = a.o; ins.b = b.o; ins.c = a.win ? lit(a.wpos, a.wlen, false) : none();
    const bool nullable = a.nullable || b.nullable;
    const int r = alloc_reg(MT_I8, nullable);
    ins.dst = r; ins.dst_nullable = nullable;
    prog->code.push_back(ins);
    Val v; v.o = none(); v.o.kind = OK_REG; v.o.idx = r; v.o.nullable = nullable;
    v.mt = MT_I8; v.dtype = B2_BOOL8; v.precision = 0; v.scale = 0; v.nullable = nullable;
    return v;
  }

  // literal re-typed to another machine type at compile time
  static bool retype_literal(Val& v, int to_mt) {
    if (v.o.kind != OK_LIT) return false;
    if (v.mt == MT_F32 || v.mt == MT_F64 || to_mt == MT_F32 || to_mt == MT_F64) {
      const bool from_int = v.mt != MT_F32 && v.mt != MT_F64;
      double d;
      if (v.mt == MT_F32) { float f; memcpy(&f, &v.o.lo, 4); d = f; }
      else if (v.mt == MT_F64) memcpy(&d, &v.o.lo, 8);
      else d = (double)(int64_t)v.o.lo;
      // an integer goes to float in one rounding, as the column path's cvt.rn.f32.s64 does: through double it would be
      // rounded twice (2^54 + 2^30 + 1 would become 2^54 instead of 2^54 + 2^31)
      if (to_mt == MT_F32) { float f = from_int ? (float)(int64_t)v.o.lo : (float)d; v.o.lo = 0; memcpy(&v.o.lo, &f, 4); v.o.hi = 0; }
      else if (to_mt == MT_F64) { memcpy(&v.o.lo, &d, 8); v.o.hi = 0; }
      else return false;
    } else {
      // integer widening/narrowing keeps the two's complement value (already sign-extended)
    }
    v.mt = to_mt;
    return true;
  }

  Val widen_int(Val v, int to_mt) {  // integer machine type change (sign extending / truncating)
    if (v.mt == to_mt) return v;
    if (v.o.kind == OK_LIT) { retype_literal(v, to_mt); return v; }
    return emit(V_CAST, v.mt, to_mt, to_mt, v.nullable, 0, &v, nullptr, nullptr, v.dtype, v.precision, v.scale);
  }

  // bring a decimal (or integral literal/column) to decimal(precision, scale) in machine type of that precision
  Val to_decimal(Val v, int precision, int scale, bool check) {
    int target_dt = decimal_dtype_for(precision);
    int target_mt = mt_of(target_dt);
    int from_scale = is_decimal(v.dtype) ? v.scale : 0;
    int from_prec = is_decimal(v.dtype) ? v.precision : default_precision(v.dtype);
    if (v.mt == MT_F32 || v.mt == MT_F64) throw Error(B2_ERR_UNSUPPORTED, "float -> decimal cast is not supported");
    if (v.o.kind == OK_LIT && !v.o.lit_null && scale >= from_scale && scale - from_scale <= 18) {
      // fold literal rescaling at compile time (GpuLiteral arithmetic is constant-folded by Catalyst too).  A value that
      // cannot take the next factor of 10 within `precision` digits is out of range: it is not folded, and the
      // instructions below turn it into NULL at run time.  Checking before each multiply keeps x below 10^38.
      __int128 x = ((__int128)v.o.hi << 64) | (unsigned __int128)(uint64_t)v.o.lo;
      __int128 lim = 1; for (int t = 0; t < precision; t++) lim *= 10;
      bool fits = true;
      for (int t = 0; t < scale - from_scale && fits; t++) {
        if (x > lim / 10 || x < -(lim / 10)) fits = false;
        else x *= 10;
      }
      if (fits && x < lim && x > -lim) {
        Val r = v;
        r.o.lo = (int64_t)(uint64_t)x; r.o.hi = (int64_t)(x >> 64);
        r.mt = target_mt; r.dtype = target_dt; r.precision = precision; r.scale = scale;
        return r;
      }
    }
    Val cur = v;
    if (scale >= from_scale) {
      cur = widen_int(cur, target_mt >= cur.mt ? target_mt : cur.mt);
      int ds = scale - from_scale;
      if (ds > 0) {
        // 10^ds * x can only leave the machine type when its digits exceed what the type holds
        int max_digits = cur.mt == MT_I32 ? 9 : (cur.mt == MT_I64 ? 18 : 38);
        bool may_overflow = from_prec + ds > max_digits;
        cur = emit(V_RESCALE_UP, cur.mt, cur.mt, cur.mt, cur.nullable || may_overflow, ds, &cur, nullptr, nullptr,
                   target_dt, precision, scale);
      }
      if (cur.mt != target_mt) {
        // narrowing truncates: check the precision on the wide value, before the cast can wrap it into range
        if (check && precision - scale < from_prec - from_scale)
          cur = emit(V_CHECK_PREC, cur.mt, cur.mt, cur.mt, true, precision, &cur, nullptr, nullptr, target_dt, precision, scale);
        check = false;
        cur = widen_int(cur, target_mt);
      }
    } else {
      int ds = from_scale - scale;
      cur = emit(V_RESCALE_DOWN, cur.mt, cur.mt, cur.mt, cur.nullable, ds, &cur, nullptr, nullptr, target_dt, precision, scale);
      // after rounding the value has at most from_prec - ds + 1 digits
      if (target_mt < cur.mt) {
        if (check && precision < from_prec - ds + 1)
          cur = emit(V_CHECK_PREC, cur.mt, cur.mt, cur.mt, true, precision, &cur, nullptr, nullptr, target_dt, precision, scale);
        check = false;
      }
      cur = widen_int(cur, target_mt);
    }
    // HALF_UP rounding on a scale decrease can carry into one more integer digit
    if (check && (precision - scale) < (from_prec - from_scale) + (scale < from_scale ? 1 : 0))
      cur = emit(V_CHECK_PREC, cur.mt, cur.mt, cur.mt, true, precision, &cur, nullptr, nullptr, target_dt, precision, scale);
    cur.dtype = target_dt; cur.precision = precision; cur.scale = scale;
    return cur;
  }

  Val compile(Expr* e) {
    if (e->op == 0) {  // GpuBoundReference
      Val v; v.o = none(); v.o.kind = OK_COL; v.o.idx = e->column; v.o.nullable = e->nullable;
      // strings can only pass through (group-by keys / filter payload); they never enter the VM
      v.mt = e->dtype == B2_STRING ? MT_I8 : mt_of(e->dtype);
      v.dtype = e->dtype; v.precision = e->precision; v.scale = e->scale; v.nullable = e->nullable;
      if (e->column >= VM_MAX_COLS) throw Error(B2_ERR_UNSUPPORTED, "too many input columns");
      if ((int)prog->col_dtype.size() <= e->column) prog->col_dtype.resize(e->column + 1, -1);
      if (prog->col_dtype[e->column] >= 0 && prog->col_dtype[e->column] != e->dtype)
        throw Error(B2_ERR_INVALID, "column bound with two different types");
      prog->col_dtype[e->column] = e->dtype;
      return v;
    }
    if (e->op == -1 && e->dtype == B2_STRING) {  // string GpuLiteral: bytes go to the program's literal pool
      Val v; v.o = lit(intern(e->str), (int64_t)e->str.size(), e->lit_null);
      v.mt = MT_I8; v.dtype = B2_STRING; v.precision = 0; v.scale = 0; v.nullable = e->lit_null;
      return v;
    }
    if (e->op == -1 && e->dtype < 0) {  // untyped NULL (CASE without ELSE): takes the type of its sibling in unify()
      Val v; v.o = lit(0, 0, true); v.mt = MT_I8; v.dtype = -1; v.precision = 0; v.scale = 0; v.nullable = true;
      return v;
    }
    if (e->op == -1) {  // GpuLiteral
      Val v; v.o = lit(e->lit_lo, e->lit_hi, e->lit_null);
      v.mt = mt_of(e->dtype); v.dtype = e->dtype; v.precision = e->precision; v.scale = e->scale; v.nullable = e->lit_null;
      return v;
    }
    if (e->op == -2) return compile_cast(e);
    switch (e->op) {
      case B2_OP_ADD: case B2_OP_SUB: case B2_OP_MUL: case B2_OP_DIV: case B2_OP_MOD: case B2_OP_PMOD:
        return compile_arith(e);
      case B2_OP_EQ: case B2_OP_NE: case B2_OP_LT: case B2_OP_LE: case B2_OP_GT: case B2_OP_GE: case B2_OP_EQ_NULLSAFE:
        return compile_compare(e);
      case B2_OP_AND: case B2_OP_OR: {
        Val a = compile(e->kids[0]), b = compile(e->kids[1]);
        if (a.dtype != B2_BOOL8 || b.dtype != B2_BOOL8) throw Error(B2_ERR_INVALID, "AND/OR need boolean operands");
        if (a.o.kind == OK_LIT) std::swap(a, b);
        if (e->op == B2_OP_AND && !a.nullable && !b.nullable && !prog->code.empty()) {
          // conjunct fusion: acc AND (x cmp y) in one pass when the comparison was the instruction just emitted
          // and feeds only this AND (its register dies here)
          const VMInstr& last = prog->code.back();
          if (a.o.kind == OK_REG && a.o.idx == last.dst && !(b.o.kind == OK_REG && b.o.idx == last.dst)) std::swap(a, b);
          const bool cmp = last.op >= V_EQ && last.op <= V_GE && !last.dst_nullable;
          if (cmp && b.o.kind == OK_REG && b.o.idx == last.dst && a.o.kind != OK_LIT && !(a.o.kind == OK_REG && a.o.idx == last.dst)) {
            static const int truth[6] = {2, 5, 1, 3, 4, 6};   // EQ NE LT LE GT GE over {<, ==, >}
            VMInstr ins = last;
            ins.aux = truth[last.op - V_EQ];
            ins.op = V_ANDCMP;
            ins.c = a.o;
            prog->code.pop_back();
            release(a); release(b);
            const int r = alloc_reg(MT_I8, false);
            ins.dst = r; ins.dst_nullable = 0;
            prog->code.push_back(ins);
            Val v; v.o = none(); v.o.kind = OK_REG; v.o.idx = r; v.o.nullable = 0;
            v.mt = MT_I8; v.dtype = B2_BOOL8; v.precision = 0; v.scale = 0; v.nullable = false;
            return v;
          }
        }
        return emit(e->op == B2_OP_AND ? V_AND : V_OR, MT_I8, MT_I8, MT_I8, a.nullable || b.nullable, 0, &a, &b, nullptr, B2_BOOL8, 0, 0);
      }
      case B2_OP_NOT: {
        Val a = compile(e->kids[0]);
        if (a.dtype != B2_BOOL8) throw Error(B2_ERR_INVALID, "NOT needs a boolean operand");
        return emit(V_NOT, MT_I8, MT_I8, MT_I8, a.nullable, 0, &a, nullptr, nullptr, B2_BOOL8, 0, 0);
      }
      case B2_OP_IS_NULL: case B2_OP_IS_NOT_NULL: {
        Val a = compile(e->kids[0]);
        return emit(e->op == B2_OP_IS_NULL ? V_ISNULL : V_ISNOTNULL, a.mt, MT_I8, MT_I8, false, 0, &a, nullptr, nullptr, B2_BOOL8, 0, 0);
      }
      case B2_OP_NEG: case B2_OP_ABS: {
        Val a = compile(e->kids[0]);
        return emit(e->op == B2_OP_NEG ? V_NEG : V_ABS, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, a.precision, a.scale);
      }
      case B2_OP_COALESCE: {
        Val a = compile(e->kids[0]), b = compile(e->kids[1]);
        unify(a, b);
        return emit(V_COALESCE, a.mt, a.mt, a.mt, a.nullable && b.nullable, 0, &a, &b, nullptr, a.dtype, a.precision, a.scale);
      }
      case B2_OP_IF: {
        Val p = compile(e->kids[0]), a = compile(e->kids[1]), b = compile(e->kids[2]);
        if (p.dtype != B2_BOOL8) throw Error(B2_ERR_INVALID, "IF needs a boolean predicate");
        unify(a, b);
        return emit(V_IF, a.mt, a.mt, a.mt, a.nullable || b.nullable, 0, &p, &a, &b, a.dtype, a.precision, a.scale);
      }
      case B2_OP_NORMALIZE_NAN_ZERO: {
        Val a = compile(e->kids[0]);
        if (!is_float(a.dtype)) return a;
        return emit(V_NORM_NAN_ZERO, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, 0, 0);
      }
      case B2_OP_SUBSTRING: {   // stringFunctions.scala:524 GpuSubstring with literal pos / len
        Val a = compile(e->kids[0]);
        if (a.dtype != B2_STRING || a.o.kind != OK_COL || a.win) throw Error(B2_ERR_UNSUPPORTED, "Substring needs a plain STRING column");
        a.win = true; a.wpos = e->lit_lo; a.wlen = e->lit_hi;
        return a;
      }
      case B2_OP_STARTS_WITH: case B2_OP_ENDS_WITH: case B2_OP_CONTAINS: case B2_OP_LIKE: {
        Val a = compile(e->kids[0]), b = compile(e->kids[1]);
        // GpuBinaryExpressionArgsAnyScalar: the right side is a scalar (stringFunctions.scala:163,189,396,972)
        if (a.dtype != B2_STRING || b.dtype != B2_STRING || b.o.kind != OK_LIT) throw Error(B2_ERR_UNSUPPORTED, "string predicate needs (STRING column, STRING literal)");
        const int kind = e->op == B2_OP_STARTS_WITH ? SP_STARTS : e->op == B2_OP_ENDS_WITH ? SP_ENDS : e->op == B2_OP_CONTAINS ? SP_CONTAINS : SP_LIKE;
        return emit_strpred(kind, a, b, e->escape);
      }
      case B2_OP_YEAR: {
        Val a = compile(e->kids[0]);
        if (a.dtype != B2_DATE32) throw Error(B2_ERR_UNSUPPORTED, "YEAR needs a date");
        return emit(V_YEAR, MT_I32, MT_I32, MT_I32, a.nullable, 0, &a, nullptr, nullptr, B2_INT32, 0, 0);
      }
    }
    throw Error(B2_ERR_UNSUPPORTED, "expression op " + std::to_string(e->op) + " is not supported");
  }

  void unify(Val& a, Val& b) {
    if (a.dtype < 0 && b.dtype < 0) throw Error(B2_ERR_INVALID, "cannot type an expression whose branches are all untyped NULL");
    if (a.dtype < 0) { a.dtype = b.dtype; a.precision = b.precision; a.scale = b.scale; a.mt = b.mt; return; }
    if (b.dtype < 0) { b.dtype = a.dtype; b.precision = a.precision; b.scale = a.scale; b.mt = a.mt; return; }
    if (a.dtype == B2_STRING || b.dtype == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "string-valued expressions (only string predicates are compiled)");
    if (is_decimal(a.dtype) && is_decimal(b.dtype)) {
      int s = std::max(a.scale, b.scale);
      int p = std::max(a.precision - a.scale, b.precision - b.scale) + s;
      if (p > 38) throw Error(B2_ERR_UNSUPPORTED, "decimal operands too wide to unify");
      a = to_decimal(a, p, s, false); b = to_decimal(b, p, s, false);
      return;
    }
    if (a.dtype != b.dtype) throw Error(B2_ERR_INVALID, "operand types differ: " + std::to_string(a.dtype) + " vs " + std::to_string(b.dtype));
  }

  Val compile_compare(Expr* e) {
    Val a = compile(e->kids[0]), b = compile(e->kids[1]);
    if (a.dtype == B2_STRING || b.dtype == B2_STRING) {   // predicates.scala:155-331 over strings: UTF8String byte order
      if (a.dtype != b.dtype) throw Error(B2_ERR_INVALID, "comparison of a string with a non-string");
      if (e->op == B2_OP_EQ_NULLSAFE) throw Error(B2_ERR_UNSUPPORTED, "<=> over strings");
      int kind = SP_EQ + (e->op - B2_OP_EQ);
      if (a.o.kind == OK_LIT && b.o.kind != OK_LIT) {
        std::swap(a, b);
        switch (kind) { case SP_LT: kind = SP_GT; break; case SP_LE: kind = SP_GE; break; case SP_GT: kind = SP_LT; break; case SP_GE: kind = SP_LE; break; }
      }
      return emit_strpred(kind, a, b, 0);
    }
    unify(a, b);
    int op = V_EQ + (e->op - B2_OP_EQ);
    if (a.o.kind == OK_LIT && b.o.kind != OK_LIT) {  // keep the literal on the right
      std::swap(a, b);
      switch (op) { case V_LT: op = V_GT; break; case V_LE: op = V_GE; break; case V_GT: op = V_LT; break; case V_GE: op = V_LE; break; }
    }
    bool nullable = (a.nullable || b.nullable) && op != V_EQNS;
    return emit(op, a.mt, MT_I8, MT_I8, nullable, 0, &a, &b, nullptr, B2_BOOL8, 0, 0);
  }

  // a +- b into DECIMAL(38, rs) when the operands' scales differ.  Rescaling the lower-scale side l first can leave 128
  // bits while the sum is still in range (|l * 10^ds| near 1.5e38, |h| near -0.9e38).  Instead the higher-scale side is
  // split as h = hq * 10^ds + hr (HALF_UP, |hr| <= 10^ds / 2) and the sum is (l +- hq) * 10^ds +- hr: l +- hq cannot
  // overflow, and a product that leaves 128 bits is at least 10^38 away from fitting anyway.
  Val capped_add_mixed(Val a, Val b, bool sub, int rs) {
    const bool a_low = a.scale < b.scale;
    const int ds = rs - std::min(a.scale, b.scale);
    a = to_decimal(a, 38, a.scale, false); b = to_decimal(b, 38, b.scale, false);
    if (a.o.kind == OK_LIT) a = emit(V_MOV, MT_I128, MT_I128, MT_I128, a.nullable, 0, &a, nullptr, nullptr, a.dtype, 38, a.scale);
    if (b.o.kind == OK_LIT) b = emit(V_MOV, MT_I128, MT_I128, MT_I128, b.nullable, 0, &b, nullptr, nullptr, b.dtype, 38, b.scale);
    Val h = a_low ? b : a, l = a_low ? a : b;
    const int D = B2_DECIMAL128, I = MT_I128;
    pin(h, true);
    Val hq = emit(V_RESCALE_DOWN, I, I, I, h.nullable, ds, &h, nullptr, nullptr, D, 38, l.scale);
    pin(hq, true);
    Val t = emit(V_RESCALE_UP, I, I, I, hq.nullable, ds, &hq, nullptr, nullptr, D, 38, rs);
    pin(h, false);
    Val hr = emit(V_SUB, I, I, I, h.nullable || t.nullable, 0, &h, &t, nullptr, D, 38, rs);
    pin(hq, false);
    // add: (l + hq) 10^ds + hr;  a - b with a low: (l - hq) 10^ds - hr;  a - b with b low: (hq - l) 10^ds + hr
    const bool un = l.nullable || hq.nullable;
    Val u = (sub && !a_low) ? emit(V_SUB, I, I, I, un, 0, &hq, &l, nullptr, D, 38, l.scale)
                            : emit(sub ? V_SUB : V_ADD, I, I, I, un, 0, &l, &hq, nullptr, D, 38, l.scale);
    Val w = emit(V_RESCALE_UP, I, I, I, true, ds, &u, nullptr, nullptr, D, 38, rs);
    Val r = emit(sub && a_low ? V_SUB : V_ADD, I, I, I, true, 0, &w, &hr, nullptr, D, 38, rs);
    return emit(V_CHECK_PREC, I, I, I, true, 38, &r, nullptr, nullptr, D, 38, rs);
  }

  Val compile_arith(Expr* e) {
    Val a = compile(e->kids[0]), b = compile(e->kids[1]);
    int vop = V_ADD + (e->op - B2_OP_ADD);
    if (is_decimal(a.dtype) || is_decimal(b.dtype)) {
      if (!is_decimal(a.dtype)) a = to_decimal(a, default_precision(a.dtype), 0, false);
      if (!is_decimal(b.dtype)) b = to_decimal(b, default_precision(b.dtype), 0, false);
      int p1 = a.precision, s1 = a.scale, p2 = b.precision, s2 = b.scale;
      if (e->op == B2_OP_ADD || e->op == B2_OP_SUB) {
        int s = std::max(s1, s2);
        int p = std::max(p1 - s1, p2 - s2) + s + 1;
        int rp = p, rs = s;
        adjust_precision_scale(rp, rs);
        if (rs != s) throw Error(B2_ERR_UNSUPPORTED, "decimal add with precision loss is not supported");
        bool capped = p > 38;
        if (capped && s1 != s2) return capped_add_mixed(a, b, e->op == B2_OP_SUB, rs);
        a = to_decimal(a, rp, rs, false); b = to_decimal(b, rp, rs, false);
        if (a.o.kind == OK_LIT && e->op == B2_OP_ADD) std::swap(a, b);
        if (a.o.kind == OK_LIT) a = emit(V_MOV, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, a.precision, a.scale);
        bool nullable = a.nullable || b.nullable || (a.mt == MT_I128 && capped);
        Val r = emit(vop, a.mt, a.mt, a.mt, nullable, 0, &a, &b, nullptr, decimal_dtype_for(rp), rp, rs);
        if (capped) r = emit(V_CHECK_PREC, r.mt, r.mt, r.mt, true, 38, &r, nullptr, nullptr, r.dtype, rp, rs);
        return r;
      }
      if (e->op == B2_OP_MUL) {
        int p = p1 + p2 + 1, s = s1 + s2;
        int rp = p, rs = s;
        adjust_precision_scale(rp, rs);
        int rdt = decimal_dtype_for(rp), rmt = mt_of(rdt);
        if (a.o.kind == OK_LIT) std::swap(a, b);
        if (a.o.kind == OK_LIT) a = emit(V_MOV, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, a.precision, a.scale);
        if (p <= 38) {
          if (rmt == MT_I128 && a.mt <= MT_I64 && b.mt <= MT_I64) {  // exact 64x64 -> 128, no widened temporaries
            a = widen_int(a, MT_I64); b = widen_int(b, MT_I64);
            return emit(V_MULW, MT_I64, MT_I128, MT_I128, a.nullable || b.nullable, 0, &a, &b, nullptr, rdt, rp, rs);
          }
          a = widen_int(a, rmt); b = widen_int(b, rmt);
          return emit(V_MUL, rmt, rmt, rmt, a.nullable || b.nullable, 0, &a, &b, nullptr, rdt, rp, rs);
        }
        if (a.mt != MT_I128 && b.mt == MT_I128) std::swap(a, b);   // the wide side goes left
        a = widen_int(a, MT_I128);
        if (b.mt != MT_I128) b = widen_int(b, MT_I64);              // 64-bit right operand: no widened temporary
        return emit(V_MULDEC, MT_I128, b.mt, MT_I128, true, s - rs, &a, &b, nullptr, B2_DECIMAL128, rp, rs);
      }
      if (e->op == B2_OP_DIV) {
        // Spark Divide: scale = max(6, s1 + p2 + 1), precision = p1 - s1 + s2 + scale (DecimalPrecision), adjusted
        int rs = std::max(6, s1 + p2 + 1), rp = p1 - s1 + s2 + rs;
        adjust_precision_scale(rp, rs);
        const int k = rs - s1 + s2;
        if (k < 0 || k > 38) throw Error(B2_ERR_UNSUPPORTED, "decimal divide with this precision/scale combination");
        if (a.o.kind == OK_LIT) a = emit(V_MOV, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, a.precision, a.scale);
        a = widen_int(a, MT_I128); b = widen_int(b, MT_I128);
        Val r = emit(V_DIVDEC, MT_I128, MT_I128, MT_I128, true, k, &a, &b, nullptr, decimal_dtype_for(rp), rp, rs);
        if (rp <= 18) r = widen_int(r, mt_of(decimal_dtype_for(rp)));
        r.dtype = decimal_dtype_for(rp); r.precision = rp; r.scale = rs;
        return r;
      }
      throw Error(B2_ERR_UNSUPPORTED, "decimal remainder is not supported yet");
    }
    if (a.dtype != b.dtype) throw Error(B2_ERR_INVALID, "arithmetic operand types differ");
    if (a.dtype == B2_BOOL8 || a.dtype == B2_STRING) throw Error(B2_ERR_INVALID, "arithmetic on non-numeric type");
    bool commut = e->op == B2_OP_ADD || e->op == B2_OP_MUL;
    if (a.o.kind == OK_LIT && commut) std::swap(a, b);
    if (a.o.kind == OK_LIT) a = emit(V_MOV, a.mt, a.mt, a.mt, a.nullable, 0, &a, nullptr, nullptr, a.dtype, a.precision, a.scale);
    // x / 0 and x % 0 are NULL; a non-zero literal divisor cannot make one
    bool div_like = (e->op == B2_OP_DIV || e->op == B2_OP_MOD || e->op == B2_OP_PMOD) && !nonzero_literal(b);
    return emit(vop, a.mt, a.mt, a.mt, a.nullable || b.nullable || div_like, 0, &a, &b, nullptr, a.dtype, 0, 0);
  }

  static bool nonzero_literal(const Val& v) {
    if (v.o.kind != OK_LIT || v.o.lit_null) return false;
    if (v.mt == MT_F32) { float f; memcpy(&f, &v.o.lo, 4); return f != 0; }
    if (v.mt == MT_F64) { double d; memcpy(&d, &v.o.lo, 8); return d != 0; }
    return v.o.lo != 0 || v.o.hi != 0;
  }
  Val int_lit(int64_t x, int mt, int dtype) {
    Val v; v.o = lit(x, x < 0 ? -1 : 0, false); v.mt = mt; v.dtype = dtype; v.precision = 0; v.scale = 0; v.nullable = false;
    return v;
  }
  void pin(const Val& v, bool on) { if (v.o.kind == OK_REG) reg_pinned[v.o.idx] = on; }

  // floorDiv(x, d) for INT64 x and a positive d: q = x / d, then IF(x % d < 0, q - 1, q)
  Val floor_div(Val x, int64_t d) {
    const int I = MT_I64;
    const Val dv = int_lit(d, I, B2_INT64), zero = int_lit(0, I, B2_INT64), one = int_lit(1, I, B2_INT64);
    pin(x, true);
    Val q = emit(V_DIV, I, I, I, x.nullable, 0, &x, &dv, nullptr, B2_INT64, 0, 0);
    pin(x, false);
    pin(q, true);
    Val r = emit(V_MOD, I, I, I, x.nullable, 0, &x, &dv, nullptr, B2_INT64, 0, 0);
    Val neg = emit(V_LT, I, MT_I8, MT_I8, r.nullable, 0, &r, &zero, nullptr, B2_BOOL8, 0, 0);
    Val qm = emit(V_SUB, I, I, I, q.nullable, 0, &q, &one, nullptr, B2_INT64, 0, 0);
    pin(q, false);
    return emit(V_IF, I, I, I, q.nullable, 0, &neg, &qm, &q, B2_INT64, 0, 0);
  }

  // GpuCast.castLongToTimestamp: seconds -> microseconds, saturating at the INT64 range
  Val seconds_to_micros(Val x) {
    const int I = MT_I64;
    const int64_t max_s = INT64_MAX / 1000000;
    const Val us = int_lit(1000000, I, B2_INT64), hi = int_lit(max_s, I, B2_INT64), lo = int_lit(-max_s, I, B2_INT64);
    const Val sat_hi = int_lit(INT64_MAX, I, B2_TIMESTAMP_US), sat_lo = int_lit(INT64_MIN, I, B2_TIMESTAMP_US);
    pin(x, true);
    Val m = emit(V_MUL, I, I, I, x.nullable, 0, &x, &us, nullptr, B2_TIMESTAMP_US, 0, 0);
    Val over = emit(V_GT, I, MT_I8, MT_I8, x.nullable, 0, &x, &hi, nullptr, B2_BOOL8, 0, 0);
    Val r1 = emit(V_IF, I, I, I, m.nullable, 0, &over, &sat_hi, &m, B2_TIMESTAMP_US, 0, 0);
    pin(x, false);
    Val under = emit(V_LT, I, MT_I8, MT_I8, x.nullable, 0, &x, &lo, nullptr, B2_BOOL8, 0, 0);
    return emit(V_IF, I, I, I, r1.nullable, 0, &under, &sat_lo, &r1, B2_TIMESTAMP_US, 0, 0);
  }

  // GpuCast.doCast for DATE32 and TIMESTAMP_US (GpuCast.scala:314-339, 370-375, 522-537).  The ABI carries no time zone, so
  // DATE <-> TIMESTAMP is refused, as are the casts Spark has no rule for (integer -> DATE, float -> TIMESTAMP).
  Val compile_datetime_cast(Val a, int to) {
    const int from = a.dtype;
    if (from == B2_DATE32) {
      if (to == B2_TIMESTAMP_US) throw Error(B2_ERR_UNSUPPORTED, "DATE -> TIMESTAMP needs a time zone");
      // date -> boolean or any number is always NULL
      Val v; v.o = lit(0, 0, true); v.mt = mt_of(to); v.dtype = to; v.precision = 0; v.scale = 0; v.nullable = true;
      return v;
    }
    if (to == B2_DATE32) throw Error(B2_ERR_UNSUPPORTED, from == B2_TIMESTAMP_US ? "TIMESTAMP -> DATE needs a time zone" : "cast to DATE from this type");
    if (from == B2_TIMESTAMP_US) {
      if (to == B2_BOOL8) return a;   // x != 0, below
      if (to == B2_FLOAT64 || to == B2_FLOAT32) {   // microseconds / 10^6 in double, then rounded to the target
        Val d = emit(V_CAST, MT_I64, MT_F64, MT_F64, a.nullable, 0, &a, nullptr, nullptr, B2_FLOAT64, 0, 0);
        double us = 1e6;
        Val dv; dv.o = lit(0, 0, false); memcpy(&dv.o.lo, &us, 8); dv.mt = MT_F64; dv.dtype = B2_FLOAT64; dv.precision = 0; dv.scale = 0; dv.nullable = false;
        Val r = emit(V_DIV, MT_F64, MT_F64, MT_F64, d.nullable, 0, &d, &dv, nullptr, B2_FLOAT64, 0, 0);
        if (to == B2_FLOAT32) r = emit(V_CAST, MT_F64, MT_F32, MT_F32, r.nullable, 0, &r, nullptr, nullptr, B2_FLOAT32, 0, 0);
        return r;
      }
      // seconds = floorDiv(microseconds, 10^6), then narrowed like any integer
      Val s = floor_div(a, 1000000);
      s = widen_int(s, mt_of(to));
      s.dtype = to;
      return s;
    }
    // to == B2_TIMESTAMP_US
    if (from == B2_FLOAT32 || from == B2_FLOAT64) throw Error(B2_ERR_UNSUPPORTED, "float -> TIMESTAMP is not supported");
    if (from == B2_BOOL8) { Val r = widen_int(a, MT_I64); r.dtype = to; return r; }   // false/true -> 0/1 microseconds
    if (from == B2_INT64) return seconds_to_micros(a);
    // byte, short, int seconds cannot overflow in microseconds
    Val w = widen_int(a, MT_I64);
    const Val us = int_lit(1000000, MT_I64, B2_INT64);
    return emit(V_MUL, MT_I64, MT_I64, MT_I64, w.nullable, 0, &w, &us, nullptr, B2_TIMESTAMP_US, 0, 0);
  }

  Val compile_cast(Expr* e) {  // GpuCast.scala:295 doCast (numeric subset)
    Val a = compile(e->kids[0]);
    int to = e->dtype;
    if (a.dtype == to && (!is_decimal(to) || (a.precision == e->precision && a.scale == e->scale))) return a;
    if (to == B2_STRING || a.dtype == B2_STRING) throw Error(B2_ERR_UNSUPPORTED, "string casts are not supported");
    if (is_decimal(to)) {
      if (a.dtype == B2_BOOL8 || a.dtype == B2_DATE32 || a.dtype == B2_TIMESTAMP_US) throw Error(B2_ERR_UNSUPPORTED, "cast to decimal from this type");
      return to_decimal(a, e->precision, e->scale, true);
    }
    if (is_decimal(a.dtype)) {
      if (to == B2_FLOAT64 || to == B2_FLOAT32) {
        Val r = emit(V_DEC2F64, a.mt, MT_F64, MT_F64, a.nullable, a.scale, &a, nullptr, nullptr, B2_FLOAT64, 0, 0);
        if (to == B2_FLOAT32) r = emit(V_CAST, MT_F64, MT_F32, MT_F32, r.nullable, 0, &r, nullptr, nullptr, B2_FLOAT32, 0, 0);
        return r;
      }
      throw Error(B2_ERR_UNSUPPORTED, "decimal -> integral cast is not supported yet");
    }
    if (a.dtype == B2_DATE32 || a.dtype == B2_TIMESTAMP_US || to == B2_DATE32 || to == B2_TIMESTAMP_US) {
      a = compile_datetime_cast(a, to);
      if (a.dtype == to) return a;
    }
    int smt = a.mt, dmt = mt_of(to);
    if (to == B2_BOOL8) {  // x != 0
      Val z; z.o = lit(0, 0, false); z.mt = smt; z.dtype = a.dtype; z.precision = 0; z.scale = 0; z.nullable = false;
      return emit(V_NE, smt, MT_I8, MT_I8, a.nullable, 0, &a, &z, nullptr, B2_BOOL8, 0, 0);
    }
    if (smt == dmt) { a.dtype = to; return a; }
    if (a.o.kind == OK_LIT && retype_literal(a, dmt)) { a.dtype = to; return a; }
    return emit(V_CAST, smt, dmt, dmt, a.nullable, 0, &a, nullptr, nullptr, to, 0, 0);
  }
};

// rows per tile: as many as fit the register budget (multiple of VM_NT, at most VM_MAX_K per thread)
void set_tile_geometry(VMProgramHeader& hdr, int bytes_per_row) {
  hdr.bytes_per_row = bytes_per_row;
  const int budget = bytes_per_row >= 24 ? VM_SMEM_BUDGET_WIDE : VM_SMEM_BUDGET;
  int k = bytes_per_row > 0 ? budget / (bytes_per_row * VM_NT) : VM_MAX_K;
  if (k > VM_MAX_K) k = VM_MAX_K;
  if (k < 1) k = 1;
  hdr.tile_rows = k * VM_NT;
  hdr.smem_bytes = bytes_per_row * hdr.tile_rows;
  if (hdr.smem_bytes > 200 * 1024) throw Error(B2_ERR_UNSUPPORTED, "expression needs too much shared memory");
}

static Program* compile_program(const b2_handle* exprs, int n) {
  if (n <= 0 || n > VM_MAX_OUTS) throw Error(B2_ERR_INVALID, "bad number of output expressions");
  std::unique_ptr<Program> prog(new Program());
  memset(&prog->hdr, 0, sizeof(prog->hdr));
  Compiler cc; cc.prog = prog.get();
  for (int i = 0; i < n; i++) {
    Val v = cc.compile(expr_from(exprs[i]));
    if (v.win) throw Error(B2_ERR_UNSUPPORTED, "Substring as a projected output: use b2_substring on the column");
    if (v.dtype < 0) throw Error(B2_ERR_INVALID, "untyped NULL output");
    if (v.dtype == B2_STRING && v.o.kind != OK_COL) throw Error(B2_ERR_UNSUPPORTED, "string literal as a projected output");
    if (v.o.kind == OK_REG) cc.reg_pinned[v.o.idx] = true;  // outputs stay live
    if (i == 0) prog->hdr.npred = (int)prog->code.size();
    prog->hdr.outs[i] = v.o;
    prog->hdr.out_mt[i] = (uint8_t)v.mt;
    prog->out_dtype.push_back(v.dtype); prog->out_scale.push_back(v.scale); prog->out_precision.push_back(v.precision);
    prog->out_nullable.push_back(v.nullable);
  }
  if (prog->code.size() > (size_t)VM_SMEM_CODE) throw Error(B2_ERR_UNSUPPORTED, "expression list compiles to more than 64 instructions; split the projection");
  prog->hdr.ninstr = (int)prog->code.size();
  prog->hdr.nregs = (int)cc.reg_width.size();
  prog->hdr.ncols = (int)prog->col_dtype.size();
  prog->hdr.nouts = n;
  set_tile_geometry(prog->hdr, cc.bump);
  prog->d_hdr = DevBuf(sizeof(VMProgramHeader));
  h2d(prog->d_hdr.p, &prog->hdr, 1);
  prog->d_code = DevBuf(std::max<size_t>(1, prog->code.size()) * sizeof(VMInstr));
  if (!prog->code.empty()) h2d(prog->d_code.p, prog->code.data(), prog->code.size());
  sync();
  return prog.release();
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_expr_column(int32_t index, int32_t dtype, int32_t precision, int32_t scale, int32_t nullable, b2_handle* out) {
  B2_TRY
  B2_CHECK(index >= 0, "negative column index");
  Expr* e = new Expr();
  e->op = 0; e->column = index; e->dtype = dtype; e->precision = precision; e->scale = scale; e->nullable = nullable != 0;
  *out = to_handle(e);
  B2_CATCH
}

int b2_expr_literal(int32_t dtype, int32_t precision, int32_t scale, const void* value16, int32_t is_null, b2_handle* out) {
  B2_TRY
  Expr* e = new Expr();
  e->op = -1; e->dtype = dtype; e->precision = precision; e->scale = scale; e->lit_null = is_null != 0; e->nullable = is_null != 0;
  if (value16) { memcpy(&e->lit_lo, value16, 8); memcpy(&e->lit_hi, (const char*)value16 + 8, 8); }
  *out = to_handle(e);
  B2_CATCH
}

static Expr* make_node(int op, std::initializer_list<b2_handle> kids) {
  std::unique_ptr<Expr> e(new Expr());
  e->op = op;
  for (auto h : kids) { Expr* k = expr_from(h); k->refs.fetch_add(1); e->kids.push_back(k); }
  return e.release();
}

int b2_expr_unary(int32_t op, b2_handle child, b2_handle* out) {
  B2_TRY
  *out = to_handle(make_node(op, {child}));
  B2_CATCH
}
int b2_expr_binary(int32_t op, b2_handle l, b2_handle r, b2_handle* out) {
  B2_TRY
  *out = to_handle(make_node(op, {l, r}));
  B2_CATCH
}
int b2_expr_ternary(int32_t op, b2_handle a, b2_handle b, b2_handle c, b2_handle* out) {
  B2_TRY
  *out = to_handle(make_node(op, {a, b, c}));
  B2_CATCH
}
int b2_expr_cast(b2_handle child, int32_t dtype, int32_t precision, int32_t scale, b2_handle* out) {
  B2_TRY
  Expr* e = make_node(-2, {child});
  e->dtype = dtype; e->precision = precision; e->scale = scale;
  *out = to_handle(e);
  B2_CATCH
}
int b2_expr_string_literal(const char* utf8, int32_t len, int32_t is_null, b2_handle* out) {
  B2_TRY
  B2_CHECK(len >= 0, "negative string length");
  Expr* e = new Expr();
  e->op = -1; e->dtype = B2_STRING; e->lit_null = is_null != 0; e->nullable = is_null != 0;
  if (utf8 && len) e->str.assign(utf8, (size_t)len);
  *out = to_handle(e);
  B2_CATCH
}
int b2_expr_like(b2_handle child, b2_handle pattern_literal, int32_t escape_char, b2_handle* out) {
  B2_TRY
  Expr* e = make_node(B2_OP_LIKE, {child, pattern_literal});
  e->escape = escape_char;
  *out = to_handle(e);
  B2_CATCH
}
int b2_expr_substring(b2_handle child, int32_t pos, int32_t len, b2_handle* out) {
  B2_TRY
  Expr* e = make_node(B2_OP_SUBSTRING, {child});
  e->lit_lo = pos; e->lit_hi = len;
  *out = to_handle(e);
  B2_CATCH
}
// GpuInSet / In over literals (GpuInSet.scala): Kleene OR of equalities — NULL input -> NULL, no match with a NULL in the
// list -> NULL, exactly Spark's In
int b2_expr_in(b2_handle child, const b2_handle* literals, int32_t n, b2_handle* out) {
  B2_TRY
  B2_CHECK(n >= 0 && n <= 24, "IN list of 0..24 literals");
  Expr* acc = nullptr;
  for (int i = 0; i < n; i++) {
    Expr* eq = make_node(B2_OP_EQ, {child, literals[i]});
    if (!acc) acc = eq;
    else {
      std::unique_ptr<Expr> o(new Expr());
      o->op = B2_OP_OR; o->kids.push_back(acc); o->kids.push_back(eq);   // takes over both references
      acc = o.release();
    }
  }
  if (!acc) {  // x IN () is false for non-null x, NULL for NULL x:  x IS NULL AND NULL  ->  (x <> x)
    acc = make_node(B2_OP_NE, {child, child});
  }
  *out = to_handle(acc);
  B2_CATCH
}
// GpuCaseWhen (conditionalExpressions.scala:322): the first branch whose condition is TRUE; NULL/false conditions fall
// through; no ELSE = NULL.  Compiled as nested GpuIf (all VM ops are side-effect free outside ANSI mode).
int b2_expr_case_when(const b2_handle* conds, const b2_handle* values, int32_t n, b2_handle else_value, b2_handle* out) {
  B2_TRY
  B2_CHECK(n >= 1 && n <= 16, "CASE WHEN with 1..16 branches");
  Expr* tail;
  if (else_value) { tail = expr_from(else_value); tail->refs.fetch_add(1); }
  else { tail = new Expr(); tail->op = -1; tail->dtype = -1; tail->lit_null = true; tail->nullable = true; }
  for (int i = n - 1; i >= 0; i--) {
    std::unique_ptr<Expr> f(new Expr());
    f->op = B2_OP_IF;
    Expr* c = expr_from(conds[i]); c->refs.fetch_add(1);
    Expr* v = expr_from(values[i]); v->refs.fetch_add(1);
    f->kids.push_back(c); f->kids.push_back(v); f->kids.push_back(tail);
    tail = f.release();
  }
  *out = to_handle(tail);
  B2_CATCH
}

int b2_expr_close(b2_handle h) {
  B2_TRY
  Expr* e = expr_from(h);
  if (e->refs.fetch_sub(1) == 1) delete e;
  B2_CATCH
}

int b2_expr_type(b2_handle h, int32_t* dtype, int32_t* precision, int32_t* scale, int32_t* nullable) {
  B2_TRY
  // type inference = compile into a scratch program and read the output descriptor
  b2_handle hs[1] = {h};
  std::unique_ptr<Program> p(compile_program(hs, 1));
  *dtype = p->out_dtype[0]; *precision = p->out_precision[0]; *scale = p->out_scale[0]; *nullable = p->out_nullable[0];
  B2_CATCH
}

int b2_program_compile(const b2_handle* exprs, int32_t nexprs, b2_handle* out) {
  B2_TRY
  *out = to_handle(compile_program(exprs, nexprs));
  B2_CATCH
}
int b2_program_info(b2_handle program, int32_t* ninstr, int32_t* nregs, int32_t* bytes_per_row, int32_t* tile_rows) {
  B2_TRY
  const Program* p = program_from(program);
  *ninstr = p->hdr.ninstr; *nregs = p->hdr.nregs; *bytes_per_row = p->hdr.bytes_per_row; *tile_rows = p->hdr.tile_rows;
  B2_CATCH
}
int b2_program_close(b2_handle h) {
  B2_TRY
  delete program_from(h);
  B2_CATCH
}

}  // extern "C"
