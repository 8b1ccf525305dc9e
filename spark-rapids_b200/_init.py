"""spark_rapids_b200 — Python host binding over the C ABI of libb200sql.so.

The product is the CUDA library; this module is (a) the ctypes binding used by tests/bench and
(b) the host-side mirror of the reference's operator interface (see execs.py).  There is no CPU
implementation here: every operation goes to the library, which fails loudly without a GPU."""
import ctypes
import numpy as np

from ._lib import lib, check, B2Error, B2ColumnInfo, B2AggSpec, B2OrderByArg, B2HostColumn, B2WindowSpec, parse_header, LIB_PATH  # noqa: F401

# b2_dtype
BOOL8, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIMESTAMP_US, DECIMAL32, DECIMAL64, DECIMAL128, STRING = range(13)
DTYPE_NAMES = ["bool8", "int8", "int16", "int32", "int64", "float32", "float64", "date32", "timestamp_us",
               "decimal32", "decimal64", "decimal128", "string"]
_NP = {BOOL8: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, FLOAT32: np.float32,
       FLOAT64: np.float64, DATE32: np.int32, TIMESTAMP_US: np.int64, DECIMAL32: np.int32, DECIMAL64: np.int64}

# b2_expr_op
OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_MOD, OP_PMOD, OP_NEG, OP_ABS = 1, 2, 3, 4, 5, 6, 7, 8
OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_EQ_NULLSAFE = 10, 11, 12, 13, 14, 15, 16
OP_AND, OP_OR, OP_NOT = 20, 21, 22
OP_IS_NULL, OP_IS_NOT_NULL, OP_COALESCE, OP_IF = 30, 31, 32, 33
OP_NORMALIZE_NAN_ZERO, OP_YEAR = 41, 42
OP_STARTS_WITH, OP_ENDS_WITH, OP_CONTAINS, OP_LIKE, OP_SUBSTRING = 50, 51, 52, 53, 54
# b2_agg_kind
AGG_SUM, AGG_COUNT, AGG_MIN, AGG_MAX, AGG_COUNT_ALL = 1, 2, 3, 4, 5
# b2_window_kind, b2_frame_type
WIN_ROW_NUMBER, WIN_RANK, WIN_DENSE_RANK, WIN_LEAD, WIN_LAG = 1, 2, 3, 4, 5
WIN_SUM, WIN_COUNT, WIN_COUNT_ALL, WIN_MIN, WIN_MAX = 10, 11, 12, 13, 14
WIN_FIRST, WIN_LAST, WIN_NTH_VALUE = 15, 16, 17
FRAME_ROWS, FRAME_RANGE, FRAME_RANGE_VALUE = 0, 1, 2
UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING = -2**63, 2**63 - 1
# b2_join_kind
JOIN_INNER, JOIN_LEFT_OUTER, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI, JOIN_FULL_OUTER, JOIN_RIGHT_OUTER = 0, 1, 2, 3, 4, 5


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def is_decimal(dt):
    return dt in (DECIMAL32, DECIMAL64, DECIMAL128)


def pack_bits(valid):
    """bool array -> Arrow LSB-first bitmask bytes"""
    return np.packbits(np.asarray(valid, dtype=bool), bitorder="little")


def unpack_bits(buf, n):
    return np.unpackbits(buf, bitorder="little")[:n].astype(bool)


def ints_to_i128(vals):
    """python ints -> (n, 2) uint64 little-endian two's complement"""
    out = np.zeros((len(vals), 2), dtype=np.uint64)
    for i, v in enumerate(vals):
        v = int(v) & ((1 << 128) - 1)
        out[i, 0] = v & 0xFFFFFFFFFFFFFFFF
        out[i, 1] = v >> 64
    return out


def i128_to_ints(arr):
    out = []
    for lo, hi in arr.reshape(-1, 2):
        v = (int(hi) << 64) | int(lo)
        if v >= 1 << 127:
            v -= 1 << 128
        out.append(v)
    return out


class Column:
    """ai.rapids.cudf.ColumnVector analogue: owns one reference on a native column."""

    def __init__(self, handle):
        self.h = ctypes.c_int64(handle)

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_column_close(self.h)
            self.h = ctypes.c_int64(0)

    # ---- construction
    @staticmethod
    def from_numpy(values, dtype=None, valid=None, scale=0):
        values = np.asarray(values)
        if dtype is None:
            dtype = {np.dtype(np.bool_): BOOL8, np.dtype(np.int8): INT8, np.dtype(np.int16): INT16, np.dtype(np.int32): INT32,
                     np.dtype(np.int64): INT64, np.dtype(np.float32): FLOAT32, np.dtype(np.float64): FLOAT64}[values.dtype]
        n = len(values)
        if dtype == DECIMAL128:
            data = ints_to_i128(values) if values.ndim == 1 else np.ascontiguousarray(values, dtype=np.uint64)
        else:
            data = np.ascontiguousarray(values.astype(_NP[dtype], copy=False))
        vb = None if valid is None else np.ascontiguousarray(pack_bits(valid))
        out = ctypes.c_int64()
        check(lib.b2_column_from_host(dtype, scale, n, _ptr(data), _ptr(vb), None, ctypes.byref(out)))
        return Column(out.value)

    @staticmethod
    def from_strings(strings):
        """list of str/bytes/None"""
        valid = np.array([s is not None for s in strings], dtype=bool)
        enc = [(s.encode() if isinstance(s, str) else (s or b"")) for s in strings]
        offsets = np.zeros(len(enc) + 1, dtype=np.int32)
        if enc:
            offsets[1:] = np.cumsum([len(e) for e in enc])
        chars = np.frombuffer(b"".join(enc), dtype=np.uint8).copy() if enc else np.zeros(0, np.uint8)
        vb = None if valid.all() else np.ascontiguousarray(pack_bits(valid))
        out = ctypes.c_int64()
        check(lib.b2_column_from_host(STRING, 0, len(enc), _ptr(chars) if len(chars) else None, _ptr(vb), _ptr(offsets), ctypes.byref(out)))
        return Column(out.value)

    @staticmethod
    def from_string_buffers(chars, offsets, valid=None):
        """Arrow string buffers (uint8 chars, int32 offsets[n+1]) -> STRING column"""
        chars = np.ascontiguousarray(chars, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        vb = None if valid is None else np.ascontiguousarray(pack_bits(valid))
        out = ctypes.c_int64()
        check(lib.b2_column_from_host(STRING, 0, len(offsets) - 1, _ptr(chars) if len(chars) else None, _ptr(vb), _ptr(offsets), ctypes.byref(out)))
        return Column(out.value)

    # ---- inspection
    def info(self):
        ci = B2ColumnInfo()
        check(lib.b2_column_info_get(self.h, ctypes.byref(ci)))
        return ci

    @property
    def dtype(self):
        return self.info().dtype

    @property
    def scale(self):
        return self.info().scale

    def __len__(self):
        return self.info().size

    @property
    def null_count(self):
        return self.info().null_count

    def to_numpy(self):
        """-> (values, valid).  DECIMAL128 -> object array of python ints; STRING -> object array of bytes."""
        ci = self.info()
        n = ci.size
        vb = np.zeros((n + 7) // 8, dtype=np.uint8)
        if ci.dtype == STRING:
            offsets = np.zeros(n + 1, dtype=np.int32)
            chars = np.zeros(max(ci.data_bytes, 1), dtype=np.uint8)
            check(lib.b2_column_to_host(self.h, _ptr(chars), _ptr(vb), _ptr(offsets)))
            raw = chars.tobytes()
            vals = np.array([raw[offsets[i]:offsets[i + 1]] for i in range(n)], dtype=object)
        elif ci.dtype == DECIMAL128:
            data = np.zeros((n, 2), dtype=np.uint64)
            check(lib.b2_column_to_host(self.h, _ptr(data), _ptr(vb), None))
            vals = np.array(i128_to_ints(data), dtype=object)
        else:
            data = np.zeros(n, dtype=_NP[ci.dtype])
            check(lib.b2_column_to_host(self.h, _ptr(data), _ptr(vb), None))
            vals = data
        return vals, unpack_bits(vb, n)

    def to_pylist(self):
        vals, valid = self.to_numpy()
        dt = self.dtype
        out = []
        for v, ok in zip(vals, valid):
            if not ok:
                out.append(None)
            elif dt == BOOL8:
                out.append(bool(v))
            elif dt == STRING:
                out.append(v.decode("utf-8", "replace"))
            elif dt in (FLOAT32, FLOAT64):
                out.append(float(v))
            else:
                out.append(int(v))
        return out


class Table:
    """ai.rapids.cudf.Table analogue."""

    def __init__(self, handle):
        self.h = ctypes.c_int64(handle)

    @staticmethod
    def from_columns(cols):
        arr = (ctypes.c_int64 * len(cols))(*[c.h.value for c in cols])
        out = ctypes.c_int64()
        check(lib.b2_table_create(arr, len(cols), ctypes.byref(out)))
        return Table(out.value)

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_table_close(self.h)
            self.h = ctypes.c_int64(0)

    @property
    def num_rows(self):
        out = ctypes.c_int64()
        check(lib.b2_table_num_rows(self.h, ctypes.byref(out)))
        return out.value

    @property
    def num_columns(self):
        out = ctypes.c_int32()
        check(lib.b2_table_num_columns(self.h, ctypes.byref(out)))
        return out.value

    def column(self, i):
        out = ctypes.c_int64()
        check(lib.b2_table_column(self.h, i, ctypes.byref(out)))
        return Column(out.value)

    def columns(self):
        return [self.column(i) for i in range(self.num_columns)]

    def to_pylists(self):
        return [c.to_pylist() for c in self.columns()]

    def to_rows(self):
        cols = self.to_pylists()
        return list(zip(*cols)) if cols else []


# ------------------------------------------------------------------------------------------------
# expressions (GpuExpression trees; each node also has a neutral s-expression form used by the
# test oracle so that the same tree drives both sides)
class Expr:
    def __init__(self, handle, sexpr):
        self.h = ctypes.c_int64(handle)
        self.sexpr = sexpr

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_expr_close(self.h)
            self.h = ctypes.c_int64(0)

    def type(self):
        dt, p, s, nl = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        check(lib.b2_expr_type(self.h, ctypes.byref(dt), ctypes.byref(p), ctypes.byref(s), ctypes.byref(nl)))
        return dt.value, p.value, s.value, bool(nl.value)

    def _bin(self, op, name, other):
        other = other if isinstance(other, Expr) else (strlit(other) if isinstance(other, (str, bytes)) else lit(other))
        out = ctypes.c_int64()
        check(lib.b2_expr_binary(op, self.h, other.h, ctypes.byref(out)))
        return Expr(out.value, (name, self.sexpr, other.sexpr))

    def _un(self, op, name):
        out = ctypes.c_int64()
        check(lib.b2_expr_unary(op, self.h, ctypes.byref(out)))
        return Expr(out.value, (name, self.sexpr))

    def __add__(self, o): return self._bin(OP_ADD, "add", o)
    def __sub__(self, o): return self._bin(OP_SUB, "sub", o)
    def __mul__(self, o): return self._bin(OP_MUL, "mul", o)
    def __truediv__(self, o): return self._bin(OP_DIV, "div", o)
    def __mod__(self, o): return self._bin(OP_MOD, "mod", o)
    def pmod(self, o): return self._bin(OP_PMOD, "pmod", o)
    def __eq__(self, o): return self._bin(OP_EQ, "eq", o)
    def __ne__(self, o): return self._bin(OP_NE, "ne", o)
    def __lt__(self, o): return self._bin(OP_LT, "lt", o)
    def __le__(self, o): return self._bin(OP_LE, "le", o)
    def __gt__(self, o): return self._bin(OP_GT, "gt", o)
    def __ge__(self, o): return self._bin(OP_GE, "ge", o)
    def eq_null_safe(self, o): return self._bin(OP_EQ_NULLSAFE, "eqns", o)
    def __and__(self, o): return self._bin(OP_AND, "and", o)
    def __or__(self, o): return self._bin(OP_OR, "or", o)
    def __invert__(self): return self._un(OP_NOT, "not")
    def __neg__(self): return self._un(OP_NEG, "neg")
    def abs(self): return self._un(OP_ABS, "abs")
    def is_null(self): return self._un(OP_IS_NULL, "isnull")
    def is_not_null(self): return self._un(OP_IS_NOT_NULL, "isnotnull")
    def normalize_nan_zero(self): return self._un(OP_NORMALIZE_NAN_ZERO, "normnz")
    def year(self): return self._un(OP_YEAR, "year")
    def coalesce(self, o): return self._bin(OP_COALESCE, "coalesce", o)
    # string predicates (stringFunctions.scala:163,189,396,972) — the right side is a literal
    def startswith(self, s): return self._bin(OP_STARTS_WITH, "startswith", s if isinstance(s, Expr) else strlit(s))
    def endswith(self, s): return self._bin(OP_ENDS_WITH, "endswith", s if isinstance(s, Expr) else strlit(s))
    def contains(self, s): return self._bin(OP_CONTAINS, "contains", s if isinstance(s, Expr) else strlit(s))

    def like(self, pattern, escape="\\"):
        pat = pattern if isinstance(pattern, Expr) else strlit(pattern)
        out = ctypes.c_int64()
        check(lib.b2_expr_like(self.h, pat.h, ord(escape), ctypes.byref(out)))
        return Expr(out.value, ("like", self.sexpr, pat.sexpr, escape))

    def substr(self, pos, length=2**31 - 1):
        out = ctypes.c_int64()
        check(lib.b2_expr_substring(self.h, int(pos), int(length), ctypes.byref(out)))
        return Expr(out.value, ("substr", self.sexpr, int(pos), int(length)))

    def isin(self, values):
        lits = [v if isinstance(v, Expr) else (strlit(v) if isinstance(v, (str, bytes)) else lit(v)) for v in values]
        arr = (ctypes.c_int64 * max(len(lits), 1))(*[x.h.value for x in lits])
        out = ctypes.c_int64()
        check(lib.b2_expr_in(self.h, arr, len(lits), ctypes.byref(out)))
        return Expr(out.value, ("in", self.sexpr, [x.sexpr for x in lits]))
    __hash__ = None

    def cast(self, dtype, precision=0, scale=0):
        out = ctypes.c_int64()
        check(lib.b2_expr_cast(self.h, dtype, precision, scale, ctypes.byref(out)))
        return Expr(out.value, ("cast", self.sexpr, (dtype, precision, scale)))


def col(index, dtype, precision=0, scale=0, nullable=True):
    out = ctypes.c_int64()
    check(lib.b2_expr_column(index, dtype, precision, scale, int(nullable), ctypes.byref(out)))
    return Expr(out.value, ("col", index, (dtype, precision, scale)))


def lit(value, dtype=None, precision=0, scale=0):
    """GpuLiteral.  For decimals `value` is the UNSCALED integer."""
    if dtype is None:
        if isinstance(value, bool):
            dtype = BOOL8
        elif isinstance(value, int):
            dtype = INT32 if -2**31 <= value < 2**31 else INT64
        elif isinstance(value, float):
            dtype = FLOAT64
        else:
            raise TypeError("cannot infer literal type of %r" % (value,))
    buf = np.zeros(2, dtype=np.uint64)
    is_null = value is None
    if not is_null:
        if dtype == FLOAT64:
            buf[0] = np.array([value], dtype=np.float64).view(np.uint64)[0]
        elif dtype == FLOAT32:
            buf[0] = int(np.array([value], dtype=np.float32).view(np.uint32)[0])
        else:
            v = int(value) & ((1 << 128) - 1)
            buf[0] = v & 0xFFFFFFFFFFFFFFFF
            buf[1] = v >> 64
    out = ctypes.c_int64()
    check(lib.b2_expr_literal(dtype, precision, scale, _ptr(buf), int(is_null), ctypes.byref(out)))
    return Expr(out.value, ("lit", value, (dtype, precision, scale)))


def strlit(value):
    """GpuLiteral(StringType); value: str / bytes / None"""
    raw = None if value is None else (value.encode() if isinstance(value, str) else bytes(value))
    out = ctypes.c_int64()
    check(lib.b2_expr_string_literal(raw, len(raw) if raw else 0, int(raw is None), ctypes.byref(out)))
    return Expr(out.value, ("lit", raw, (STRING, 0, 0)))


def case_when(branches, otherwise=None):
    """GpuCaseWhen: branches = [(condition Expr, value Expr)], otherwise = Expr or None (NULL)"""
    conds = (ctypes.c_int64 * len(branches))(*[c.h.value for c, _ in branches])
    vals = (ctypes.c_int64 * len(branches))(*[v.h.value for _, v in branches])
    out = ctypes.c_int64()
    check(lib.b2_expr_case_when(conds, vals, len(branches), otherwise.h if otherwise is not None else ctypes.c_int64(0), ctypes.byref(out)))
    return Expr(out.value, ("case", [(c.sexpr, v.sexpr) for c, v in branches], otherwise.sexpr if otherwise is not None else None))


def if_else(pred, a, b):
    out = ctypes.c_int64()
    check(lib.b2_expr_ternary(OP_IF, pred.h, a.h, b.h, ctypes.byref(out)))
    return Expr(out.value, ("if", pred.sexpr, a.sexpr, b.sexpr))


class Program:
    """ast.CompiledExpression analogue: N bound expressions compiled into one fused kernel program."""

    def __init__(self, exprs):
        self.exprs = list(exprs)
        arr = (ctypes.c_int64 * len(self.exprs))(*[e.h.value for e in self.exprs])
        out = ctypes.c_int64()
        check(lib.b2_program_compile(arr, len(self.exprs), ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def info(self):
        """-> {ninstr, nregs, bytes_per_row, tile_rows}: the compiled program's geometry"""
        v = [ctypes.c_int32() for _ in range(4)]
        check(lib.b2_program_info(self.h, *[ctypes.byref(x) for x in v]))
        return dict(zip(("ninstr", "nregs", "bytes_per_row", "tile_rows"), (x.value for x in v)))

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_program_close(self.h)
            self.h = ctypes.c_int64(0)


def _agg_specs(aggs):
    """aggs: list of (kind, column, out_dtype, out_scale, out_precision)"""
    arr = (B2AggSpec * max(len(aggs), 1))()
    for i, a in enumerate(aggs):
        a = tuple(a) + (0,) * (5 - len(a))
        arr[i].kind, arr[i].column, arr[i].out_dtype, arr[i].out_scale, arr[i].out_precision = a
    return arr


def _i32s(xs):
    return (ctypes.c_int32 * max(len(xs), 1))(*xs)


def _order_args(keys):
    arr = (B2OrderByArg * max(len(keys), 1))()
    for i, k in enumerate(keys):
        arr[i].column, arr[i].ascending, arr[i].nulls_first = int(k[0]), int(k[1]), int(k[2])
    return arr


class Frame:
    """a window frame: its type and its bounds, with 0 = CURRENT ROW and None = UNBOUNDED PRECEDING (lower) / FOLLOWING (upper).
    FRAME_ROWS: bounds are row offsets.  FRAME_RANGE: only (None, 0) and (None, None).  FRAME_RANGE_VALUE: bounds are value
    offsets in the units of the single ORDER BY column (integers: values; DATE32: days; TIMESTAMP_US: microseconds; decimals:
    unscaled values at the column's scale), subtracted instead of added under a descending order; 0 is the peer group's edge"""

    def __init__(self, frame_type, lower, upper):
        self.type, self.lower, self.upper = frame_type, lower, upper


def rows(lower, upper):
    """ROWS BETWEEN lower AND upper (None = UNBOUNDED PRECEDING / FOLLOWING)"""
    return Frame(FRAME_ROWS, lower, upper)


def range_running():
    """RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW: Spark's default frame with ORDER BY"""
    return Frame(FRAME_RANGE, None, 0)


def range_between(lower, upper):
    """RANGE BETWEEN lower AND upper by value (None = UNBOUNDED PRECEDING / FOLLOWING, 0 = CURRENT ROW), e.g. 7 days before a
    DATE32 row up to it: range_between(-7, 0)"""
    return Frame(FRAME_RANGE_VALUE, lower, upper)


def unbounded():
    """the whole partition: Spark's default frame without ORDER BY"""
    return Frame(FRAME_ROWS, None, None)


class WindowFunc:
    """one window function: kind (WIN_*), its column, a Frame (aggregates, FIRST / LAST / NTH_VALUE), LEAD / LAG offset and
    default or NTH_VALUE's n (in offset), for a decimal SUM the result type (out_dtype, out_precision; the scale is the input's),
    and IGNORE NULLS for FIRST / LAST / NTH_VALUE"""

    def __init__(self, kind, column=0, frame=None, offset=1, default=None, default_dtype=None, out_dtype=0, out_precision=0,
                 ignore_nulls=False):
        self.kind, self.column, self.frame, self.offset = kind, column, frame, offset
        self.default, self.default_dtype = default, default_dtype
        self.out_dtype, self.out_precision = out_dtype, out_precision
        self.ignore_nulls = ignore_nulls


def row_number():
    return WindowFunc(WIN_ROW_NUMBER)


def rank():
    return WindowFunc(WIN_RANK)


def dense_rank():
    return WindowFunc(WIN_DENSE_RANK)


def _offset_default(default, dtype):
    if isinstance(default, float) and dtype not in (FLOAT32, FLOAT64):
        raise ValueError("a float LEAD / LAG default needs dtype=FLOAT32 or FLOAT64 (the column's type)")
    return default


def lead(column, offset=1, default=None, dtype=None):
    """dtype: the column's type, required with a float default (FLOAT32 and FLOAT64 defaults are encoded differently)"""
    return WindowFunc(WIN_LEAD, column, offset=offset, default=_offset_default(default, dtype), default_dtype=dtype)


def lag(column, offset=1, default=None, dtype=None):
    return WindowFunc(WIN_LAG, column, offset=offset, default=_offset_default(default, dtype), default_dtype=dtype)


def win_sum(column, frame, out_dtype=0, out_precision=0):
    """decimal columns: out_dtype DECIMAL64 / DECIMAL128 and out_precision (Spark: min(38, p + 10))"""
    return WindowFunc(WIN_SUM, column, frame, out_dtype=out_dtype, out_precision=out_precision)


def win_count(column, frame):
    return WindowFunc(WIN_COUNT, column, frame)


def win_count_all(frame):
    return WindowFunc(WIN_COUNT_ALL, 0, frame)


def win_min(column, frame):
    return WindowFunc(WIN_MIN, column, frame)


def win_max(column, frame):
    return WindowFunc(WIN_MAX, column, frame)


def first_value(column, frame, ignore_nulls=False):
    """first_value(column) [IGNORE NULLS] over frame: the value at the frame's first row (the first non-NULL one)"""
    return WindowFunc(WIN_FIRST, column, frame, ignore_nulls=ignore_nulls)


def last_value(column, frame, ignore_nulls=False):
    """last_value(column) [IGNORE NULLS] over frame; with rows(None, 0) and ignore_nulls, a forward fill"""
    return WindowFunc(WIN_LAST, column, frame, ignore_nulls=ignore_nulls)


def nth_value(column, n, frame, ignore_nulls=False):
    """nth_value(column, n) [IGNORE NULLS] over frame: the value at the frame's n-th row (n-th non-NULL one), n >= 1"""
    return WindowFunc(WIN_NTH_VALUE, column, frame, offset=n, ignore_nulls=ignore_nulls)


def _literal16(value, dtype):
    buf = np.zeros(2, dtype=np.uint64)
    if dtype == FLOAT32:
        buf[0] = int(np.array([value], dtype=np.float32).view(np.uint32)[0])
    elif dtype == FLOAT64:
        buf[0] = np.array([value], dtype=np.float64).view(np.uint64)[0]
    else:
        v = int(value) & ((1 << 128) - 1)
        buf[0] = v & 0xFFFFFFFFFFFFFFFF
        buf[1] = v >> 64
    return buf.view(np.uint8)


def _window_specs(funcs):
    """funcs: WindowFunc objects, or tuples (kind, column, frame, ...) of WindowFunc's arguments"""
    arr = (B2WindowSpec * max(len(funcs), 1))()
    for i, f in enumerate(funcs):
        if not isinstance(f, WindowFunc):
            f = WindowFunc(*f)
        s = arr[i]
        s.kind, s.column, s.offset = f.kind, f.column, f.offset
        fr = f.frame or Frame(FRAME_ROWS, None, 0)
        s.frame = fr.type
        s.lower = UNBOUNDED_PRECEDING if fr.lower is None else fr.lower
        s.upper = UNBOUNDED_FOLLOWING if fr.upper is None else fr.upper
        s.default_is_null = int(f.default is None)
        if f.default is not None:
            s.default_value[:] = list(_literal16(f.default, f.default_dtype))
        s.out_dtype, s.out_precision = f.out_dtype, f.out_precision
        s.ignore_nulls = int(bool(f.ignore_nulls))
    return arr


def window(table, partition_by, order_by, funcs):
    """b2_window over one batch sorted by (partition_by, order_by): the input columns, then one column per function.
    order_by: (column, ascending, nulls_first) tuples"""
    out = ctypes.c_int64()
    check(lib.b2_window(table.h, _i32s(partition_by), len(partition_by), _order_args(order_by), len(order_by), _window_specs(funcs), len(funcs),
                        ctypes.byref(out)))
    return Table(out.value)


def init(device=0, pool_bytes=0):
    check(lib.b2_init(device, pool_bytes))


def sync():
    check(lib.b2_stream_sync())


def project(program, table):
    out = ctypes.c_int64()
    check(lib.b2_project(program.h, table.h, ctypes.byref(out)))
    return Table(out.value)


def filter(program, table):  # noqa: A001 - mirrors Table.filter
    out = ctypes.c_int64()
    check(lib.b2_filter(program.h, table.h, ctypes.byref(out)))
    return Table(out.value)


def filter_select(program, table, keep_cols):
    """GpuFilterExec under a column-pruning project, fused: only keep_cols are compacted"""
    out = ctypes.c_int64()
    check(lib.b2_filter_select(program.h, table.h, _i32s(keep_cols), len(keep_cols), ctypes.byref(out)))
    return Table(out.value)


def substring(column, pos, length=2**31 - 1):
    out = ctypes.c_int64()
    check(lib.b2_substring(column.h, int(pos), int(length), ctypes.byref(out)))
    return Column(out.value)


def filter_mask(table, mask):
    out = ctypes.c_int64()
    check(lib.b2_filter_mask(table.h, mask.h, ctypes.byref(out)))
    return Table(out.value)


def filter_row_ids(program, table):
    """selection vector: INT32 ids (ascending) of the rows that pass"""
    out = ctypes.c_int64()
    check(lib.b2_filter_row_ids(program.h, table.h, ctypes.byref(out)))
    return Column(out.value)


def filter_count(program, table):
    out = ctypes.c_int64()
    check(lib.b2_filter_count(program.h, table.h, ctypes.byref(out)))
    return out.value


def reduce(table, aggs):  # noqa: A001
    out = ctypes.c_int64()
    check(lib.b2_reduce(table.h, _agg_specs(aggs), len(aggs), ctypes.byref(out)))
    return Table(out.value)


def groupby(table, keys, aggs):
    out = ctypes.c_int64()
    check(lib.b2_groupby(table.h, _i32s(keys), len(keys), _agg_specs(aggs), len(aggs), ctypes.byref(out)))
    return Table(out.value)


def scan_aggregate(program, has_predicate, table, keys, aggs):
    out = ctypes.c_int64()
    check(lib.b2_scan_aggregate(program.h, int(has_predicate), table.h, _i32s(keys), len(keys), _agg_specs(aggs), len(aggs),
                                ctypes.byref(out)))
    return Table(out.value)


def distinct_count(table, keys):
    out = ctypes.c_int64()
    check(lib.b2_distinct_count(table.h, _i32s(keys), len(keys), ctypes.byref(out)))
    return out.value


def gather(table, gather_map, nullify_oob=False):
    out = ctypes.c_int64()
    check(lib.b2_gather(table.h, gather_map.h, int(nullify_oob), ctypes.byref(out)))
    return Table(out.value)


def concat(tables):
    arr = (ctypes.c_int64 * len(tables))(*[t.h.value for t in tables])
    out = ctypes.c_int64()
    check(lib.b2_concat(arr, len(tables), ctypes.byref(out)))
    return Table(out.value)


def slice_table(table, start, end):
    out = ctypes.c_int64()
    check(lib.b2_slice(table.h, start, end, ctypes.byref(out)))
    return Table(out.value)


def kernel_launch_count():
    out = ctypes.c_int64()
    check(lib.b2_kernel_launch_count(ctypes.byref(out)))
    return out.value


class Event:
    def __init__(self):
        out = ctypes.c_int64()
        check(lib.b2_event_create(ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def record(self):
        check(lib.b2_event_record(self.h))
        return self

    def elapsed_ms(self, stop):
        ms = ctypes.c_float()
        check(lib.b2_event_elapsed_ms(self.h, stop.h, ctypes.byref(ms)))
        return ms.value

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_event_close(self.h)
            self.h = ctypes.c_int64(0)


# ---- a6/a7 joins ----------------------------------------------------------------------------------
class JoinHashTable:
    """persistent build-side hash table (built once per build batch)"""

    def __init__(self, build_keys, nulls_equal=False):
        out = ctypes.c_int64()
        check(lib.b2_join_build(build_keys.h, int(nulls_equal), ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def probe(self, probe_keys, kind=JOIN_INNER, selection=None):
        """-> (left_map Column, right_map Column|None); selection: INT32 row ids of probe_keys (filter_row_ids) that take part.
        JOIN_RIGHT_OUTER: the inner maps, then (INT32_MIN, b) for every build row b no probe row matched, ascending"""
        lm, rm = ctypes.c_int64(), ctypes.c_int64()
        check(lib.b2_join_probe_sel(self.h, probe_keys.h, selection.h if selection is not None else 0, kind, ctypes.byref(lm), ctypes.byref(rm)))
        return Column(lm.value), (Column(rm.value) if rm.value else None)

    def probe_filter(self, table, key_col, predicate):
        """INNER join of the rows of `table` that pass `predicate` (a Program), keyed on column key_col
        -> (left_map Column of original row ids, right_map Column, rows that passed the filter)"""
        lm, rm, npass = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        check(lib.b2_join_probe_filter(self.h, table.h, int(key_col), predicate.h, ctypes.byref(lm), ctypes.byref(rm), ctypes.byref(npass)))
        return Column(lm.value), Column(rm.value), npass.value

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_join_hash_table_close(self.h)
            self.h = ctypes.c_int64(0)


class JoinTracker:
    """one bit per build row of `table` (a JoinHashTable): the build rows that found a partner across probe batches, for outer
    joins that preserve the build side"""

    def __init__(self, table):
        out = ctypes.c_int64()
        check(lib.b2_join_tracker_create(table.h, ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)
        self._table = table   # the bits stand for its build rows

    def probe(self, table, probe_keys, kind=JOIN_INNER, selection=None):
        """table.probe (kind JOIN_INNER or JOIN_LEFT_OUTER) that also marks every build row it finds"""
        lm, rm = ctypes.c_int64(), ctypes.c_int64()
        check(lib.b2_join_probe_track(table.h, probe_keys.h, selection.h if selection is not None else 0, kind, self.h, ctypes.byref(lm),
                                      ctypes.byref(rm)))
        return Column(lm.value), Column(rm.value)

    def mark(self, right_map, passed=None):
        """marks right_map[i] where passed[i] (BOOL8 Column, NULL = false; None: every i); negative entries are skipped"""
        check(lib.b2_join_tracker_mark(self.h, right_map.h, passed.h if passed is not None else 0))

    def unmatched(self):
        """INT32 Column: the build rows never marked, ascending"""
        out = ctypes.c_int64()
        check(lib.b2_join_tracker_unmatched(self.h, ctypes.byref(out)))
        return Column(out.value)

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_join_tracker_close(self.h)
            self.h = ctypes.c_int64(0)


# ---- a8 sort ----------------------------------------------------------------------------------------
def sort_order(table, keys):
    """keys: [(column, ascending, nulls_first)] -> INT32 permutation column"""
    out = ctypes.c_int64()
    check(lib.b2_sort_order(table.h, _order_args(keys), len(keys), ctypes.byref(out)))
    return Column(out.value)


def order_by(table, keys):
    out = ctypes.c_int64()
    check(lib.b2_order_by(table.h, _order_args(keys), len(keys), ctypes.byref(out)))
    return Table(out.value)


def top_n(table, keys, n):
    out = ctypes.c_int64()
    check(lib.b2_top_n(table.h, _order_args(keys), len(keys), n, ctypes.byref(out)))
    return Table(out.value)


def merge_sorted(tables, keys):
    arr = (ctypes.c_int64 * len(tables))(*[t.h.value for t in tables])
    out = ctypes.c_int64()
    check(lib.b2_merge_sorted(arr, len(tables), _order_args(keys), len(keys), ctypes.byref(out)))
    return Table(out.value)


def search_bounds(sorted_table, values_table, keys, upper):
    out = ctypes.c_int64()
    check(lib.b2_search_bounds(sorted_table.h, values_table.h, _order_args(keys), len(keys), int(upper), ctypes.byref(out)))
    return Column(out.value)


# ---- a9 hash partition ------------------------------------------------------------------------------
def murmur3(table, cols, seed=42):
    out = ctypes.c_int64()
    check(lib.b2_murmur3(table.h, _i32s(cols), len(cols), seed, ctypes.byref(out)))
    return Column(out.value)


def hash_partition(table, key_cols, num_partitions, seed=42):
    """-> (partitioned Table, offsets list[num_partitions+1])"""
    out = ctypes.c_int64()
    offs = (ctypes.c_int32 * (num_partitions + 1))()
    check(lib.b2_hash_partition(table.h, _i32s(key_cols), len(key_cols), seed, num_partitions, ctypes.byref(out), offs))
    return Table(out.value), list(offs)


def hash_split(table, keys, seed, num_parts, sel=None, keep=None):
    """rows of `table` (only those the INT32 selection vector `sel` names, when given) split by pmod(murmur3(keys, seed),
    num_parts) -> list of num_parts Tables (None for an empty part) holding the columns `keep` (default all), rows in input order"""
    out = (ctypes.c_int64 * num_parts)()
    kp = None if keep is None else _i32s(keep)
    check(lib.b2_hash_split(table.h, sel.h if sel is not None else 0, _i32s(keys), len(keys), seed, num_parts, kp,
                            0 if keep is None else len(keep), out))
    return [Table(h) if h else None for h in out]


def partition_by_ids(table, part_ids, num_partitions):
    out = ctypes.c_int64()
    offs = (ctypes.c_int32 * (num_partitions + 1))()
    check(lib.b2_partition_by_ids(table.h, part_ids.h, num_partitions, ctypes.byref(out), offs))
    return Table(out.value), list(offs)


# ---- a11 rows ---------------------------------------------------------------------------------------
def table_to_rows(table):
    """-> (numpy uint8 [nrows, row_bytes])"""
    rb = ctypes.c_int32()
    check(lib.b2_rows_size(table.h, ctypes.byref(rb)))
    n = table.num_rows
    buf = np.zeros((n, rb.value), dtype=np.uint8)
    check(lib.b2_table_to_rows(table.h, _ptr(buf), buf.nbytes))
    return buf


def table_from_rows(rows, dtypes, scales=None):
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    scales = scales or [0] * len(dtypes)
    out = ctypes.c_int64()
    check(lib.b2_table_from_rows(_ptr(rows), rows.shape[0], _i32s(dtypes), _i32s(scales), len(dtypes), ctypes.byref(out)))
    return Table(out.value)


# ---- (e) exchange -----------------------------------------------------------------------------------
class Comm:
    """NCCL communicator for the shuffle exchange; the unique id is broadcast by the caller
    (torch.distributed / any rendezvous)."""

    @staticmethod
    def unique_id():
        buf = np.zeros(128, dtype=np.uint8)
        check(lib.b2_comm_unique_id(_ptr(buf)))
        return buf

    def __init__(self, unique_id, rank, world):
        uid = np.ascontiguousarray(unique_id, dtype=np.uint8)
        out = ctypes.c_int64()
        check(lib.b2_comm_init(_ptr(uid), rank, world, ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)
        self.rank, self.world = rank, world

    def exchange(self, partitioned_table, offsets):
        out = ctypes.c_int64()
        check(lib.b2_exchange(self.h, partitioned_table.h, _i32s(offsets), ctypes.byref(out)))
        return Table(out.value)

    def exchange_hash(self, table, key_cols, seed=42):
        """fused hash partition + peer-store exchange; table may be None (no batch on this rank).  -> (Table|None, any_data)"""
        out, anyd = ctypes.c_int64(), ctypes.c_int32()
        check(lib.b2_exchange_hash(self.h, table.h if table is not None else ctypes.c_int64(0), _i32s(key_cols), len(key_cols), seed,
                                   ctypes.byref(out), ctypes.byref(anyd)))
        return (Table(out.value) if out.value else None), bool(anyd.value)

    def exchange_hash_sel(self, table, key_cols, selection=None, out_cols=None, seed=42):
        """exchange_hash over the rows of `table` that the INT32 column `selection` names (all rows when None), sending only
        the columns `out_cols` (all when None); key_cols index `table` itself.  -> (Table|None, any_data)"""
        out, anyd = ctypes.c_int64(), ctypes.c_int32()
        oc = None if not out_cols else _i32s(out_cols)
        check(lib.b2_exchange_hash_sel(self.h, table.h if table is not None else ctypes.c_int64(0),
                                       selection.h if selection is not None else ctypes.c_int64(0), oc, len(out_cols or []),
                                       _i32s(key_cols), len(key_cols), seed, ctypes.byref(out), ctypes.byref(anyd)))
        return (Table(out.value) if out.value else None), bool(anyd.value)

    def fused_ready(self):
        ok = ctypes.c_int32()
        check(lib.b2_comm_fused_ready(self.h, ctypes.byref(ok)))
        return bool(ok.value)

    def stats(self):
        out = (ctypes.c_int64 * 4)()
        check(lib.b2_comm_stats(self.h, out))
        return {"bytes_sent": out[0], "bytes_received": out[1], "calls": out[2], "arena_bytes": out[3]}

    def broadcast(self, table, root):
        out = ctypes.c_int64()
        check(lib.b2_broadcast_table(self.h, table.h if table is not None else ctypes.c_int64(0), root, ctypes.byref(out)))
        return Table(out.value)

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_comm_close(self.h)
            self.h = ctypes.c_int64(0)


# ---- a10 parquet ------------------------------------------------------------------------------------
def parquet_decode(buf, columns):
    """buf: bytes / numpy uint8 holding the reassembled mini file (PAR1 ... footer len PAR1);
    columns: names in output order.  H2D copy happens inside the call."""
    arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
    names = (ctypes.c_char_p * len(columns))(*[c.encode() for c in columns])
    out = ctypes.c_int64()
    check(lib.b2_parquet_decode(_ptr(arr), arr.nbytes, names, len(columns), ctypes.byref(out)))
    return Table(out.value)


def parquet_decode_device(buf, dev_ptr, columns):
    """same, with the file bytes already resident in device memory at dev_ptr (>= 16 bytes of slack after the end)"""
    arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
    names = (ctypes.c_char_p * len(columns))(*[c.encode() for c in columns])
    out = ctypes.c_int64()
    check(lib.b2_parquet_decode_device(_ptr(arr), ctypes.c_void_p(dev_ptr), arr.nbytes, names, len(columns), ctypes.byref(out)))
    return Table(out.value)


def parquet_num_row_groups(buf):
    arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
    n = ctypes.c_int32()
    check(lib.b2_parquet_num_row_groups(_ptr(arr), arr.nbytes, ctypes.byref(n)))
    return n.value


def parquet_decode_row_groups(buf, columns, rg_begin, rg_end, dev_ptr=None):
    """one input split: decode row groups [rg_begin, rg_end) only (dev_ptr: file bytes already in HBM)"""
    arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
    names = (ctypes.c_char_p * len(columns))(*[c.encode() for c in columns])
    out = ctypes.c_int64()
    check(lib.b2_parquet_decode_row_groups(_ptr(arr), ctypes.c_void_p(dev_ptr) if dev_ptr else None, arr.nbytes, names, len(columns),
                                           int(rg_begin), int(rg_end), ctypes.byref(out)))
    return Table(out.value)


# ---- (f4) memory pressure -------------------------------------------------------------------------------
class Spillable:
    """SpillableColumnarBatch: the store may move the batch to host memory while nobody holds the table from get()"""

    def __init__(self, table):
        out = ctypes.c_int64()
        check(lib.b2_spillable_create(table.h, ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def get(self):
        out = ctypes.c_int64()
        check(lib.b2_spillable_get(self.h, ctypes.byref(out)))
        return Table(out.value)

    @property
    def spilled(self):
        v = ctypes.c_int32()
        check(lib.b2_spillable_is_spilled(self.h, ctypes.byref(v)))
        return bool(v.value)

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_spillable_close(self.h)
            self.h = ctypes.c_int64(0)

    __del__ = close


def spill(want_bytes=2**62):
    out = ctypes.c_int64()
    check(lib.b2_spill(int(want_bytes), ctypes.byref(out)))
    return out.value


def memory_stats():
    out = (ctypes.c_int64 * 6)()
    check(lib.b2_memory_stats(out))
    return {"in_use": out[0], "limit": out[1], "spilled_bytes": out[2], "unspilled_bytes": out[3], "retries": out[4], "splits": out[5]}


def set_alloc_limit(nbytes):
    check(lib.b2_set_alloc_limit(int(nbytes)))


def device_bytes_in_use():
    out = ctypes.c_int64()
    check(lib.b2_device_bytes_in_use(ctypes.byref(out)))
    return out.value


def semaphore_init(permits):
    check(lib.b2_semaphore_init(int(permits)))


def semaphore_acquire():
    check(lib.b2_semaphore_acquire())


def semaphore_release():
    check(lib.b2_semaphore_release())


def semaphore_stats():
    out = (ctypes.c_int64 * 3)()
    check(lib.b2_semaphore_stats(out))
    return {"permits": out[0], "holders": out[1], "waits": out[2]}


# ---- (f1) shuffle wire format --------------------------------------------------------------------------
def serialize_table(table, row_start=0, row_end=None):
    """GpuColumnarBatchSerializer: rows [row_start, row_end) -> bytes (numpy uint8) in the B2T1 wire format"""
    row_end = table.num_rows if row_end is None else row_end
    n = ctypes.c_int64()
    check(lib.b2_serialized_size(table.h, row_start, row_end, ctypes.byref(n)))
    buf = np.zeros(n.value, dtype=np.uint8)
    w = ctypes.c_int64()
    check(lib.b2_serialize_table(table.h, row_start, row_end, _ptr(buf), buf.nbytes, ctypes.byref(w)))
    return buf[:w.value]


def deserialize_concat(buffers):
    """GpuShuffleCoalesceExec: serialised tables -> one device Table (host concat, single upload)"""
    arrs = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else b) for b in buffers]
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    lens = (ctypes.c_int64 * len(arrs))(*[a.nbytes for a in arrs])
    out = ctypes.c_int64()
    check(lib.b2_deserialize_concat(ptrs, lens, len(arrs), ctypes.byref(out)))
    return Table(out.value)


class ParquetChunkedReader:
    """ai.rapids.cudf.ParquetChunkedReader analogue: iterate tables of <= chunk_byte_limit decoded bytes"""

    def __init__(self, buf, columns, chunk_byte_limit):
        self.arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
        names = (ctypes.c_char_p * len(columns))(*[c.encode() for c in columns])
        out = ctypes.c_int64()
        check(lib.b2_parquet_chunked_open(_ptr(self.arr), self.arr.nbytes, names, len(columns), int(chunk_byte_limit), ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def has_next(self):
        v = ctypes.c_int32()
        check(lib.b2_parquet_chunked_has_next(self.h, ctypes.byref(v)))
        return bool(v.value)

    def read_chunk(self):
        out = ctypes.c_int64()
        check(lib.b2_parquet_chunked_next(self.h, ctypes.byref(out)))
        return Table(out.value)

    def __iter__(self):
        while self.has_next():
            yield self.read_chunk()

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_parquet_chunked_close(self.h)
            self.h = ctypes.c_int64(0)

    __del__ = close


# ---- profiling / raw buffers (bench.py) ---------------------------------------------------------------
def profile_enable(on=True):
    check(lib.b2_profile_enable(int(on)))


def profile_report():
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib.b2_profile_report(buf, len(buf)))
    return json.loads(buf.value.decode())


def host_register(arr):
    check(lib.b2_host_register(_ptr(arr), arr.nbytes))


def host_unregister(arr):
    check(lib.b2_host_unregister(_ptr(arr)))


class DeviceBuffer:
    def __init__(self, nbytes):
        out = ctypes.c_void_p()
        check(lib.b2_device_alloc(nbytes, ctypes.byref(out)))
        self.ptr, self.nbytes = out.value, nbytes

    def copy_from_host(self, arr):
        check(lib.b2_memcpy_h2d(ctypes.c_void_p(self.ptr), _ptr(arr), arr.nbytes))

    def __del__(self):
        if getattr(self, "ptr", None):
            lib.b2_device_free(ctypes.c_void_p(self.ptr))
            self.ptr = None


def parquet_last_stats():
    out = (ctypes.c_int64 * 5)()
    check(lib.b2_parquet_last_stats(out))
    return {"compressed_in": out[0], "decompressed_out": out[1], "page_bytes": out[2], "column_bytes": out[3], "pages": out[4]}


class AsyncUpload:
    """pinned host buffer -> device on the copy stream (overlaps the compute stream)"""

    def __init__(self, arr):
        out = ctypes.c_int64()
        check(lib.b2_upload_start(_ptr(arr), arr.nbytes, ctypes.byref(out)))
        self.h = ctypes.c_int64(out.value)

    def wait(self):
        """order the compute stream after the copy; returns the device pointer"""
        p = ctypes.c_void_p()
        check(lib.b2_upload_wait(self.h, ctypes.byref(p)))
        return p.value

    def free(self):
        if self.h.value:
            check(lib.b2_upload_free(self.h))
            self.h = ctypes.c_int64(0)

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib.b2_upload_free(self.h)
            self.h = ctypes.c_int64(0)
