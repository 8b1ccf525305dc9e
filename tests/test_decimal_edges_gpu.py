"""Decimal arithmetic and casts of the expression VM (csrc/expr.cu compiles, csrc/vm.cuh runs) against an exact
reference written here on Python ints and decimal.Decimal.

The reference is Spark's non-ANSI decimal semantics: the result type of + - * / from DecimalPrecision with
adjustPrecisionScale (precision loss allowed), one HALF_UP rounding of the exact value to the result scale, and NULL
when the rounded value needs more than the result precision.  Casts round HALF_UP on a scale decrease and give NULL
when the value does not fit.  Decimal -> double is float(v) / float(10**s): one correctly rounded int -> double, then
one IEEE division by the correctly rounded power of ten.

Inputs are uniform in digit count, so results land on both sides of the NULL boundary, and every case appends rows
built for the edges where integer decimal kernels go wrong: HALF_UP ties and the rows just below them, results that
round to 10^38 or to 10^38 - 1, 256-bit products, quotients that leave 128 bits, and values whose rescaled form wraps
into range in a narrower machine type.  Every case runs twice: without NULLs over 2 full 4096-row tiles plus a partial
one (so both the fast and the checked row loops run), and with NULLs.
"""
import random
import struct
from decimal import ROUND_HALF_UP, Decimal, localcontext

import numpy as np
import pytest

from oracle import spark_cpu as O

pytestmark = pytest.mark.gpu

D32, D64, D128 = O.DECIMAL32, O.DECIMAL64, O.DECIMAL128
INTS = {O.INT8: 8, O.INT16: 16, O.INT32: 32, O.INT64: 64}
NP_OF = {O.INT8: np.int8, O.INT16: np.int16, O.INT32: np.int32, O.INT64: np.int64, D32: np.int32, D64: np.int64}
N_FULL = 2 * 4096 + 777   # two full tiles of any tile size (tile_rows <= 4096) and a partial one


# ---- reference -------------------------------------------------------------------------------------------------------
def dec_dtype(p):
    return D32 if p <= 9 else (D64 if p <= 18 else D128)


def round_half_up(x, k):
    """x / 10^k rounded half away from zero (k >= 0), exactly"""
    if k == 0:
        return x
    with localcontext() as c:
        c.prec = 200
        c.rounding = ROUND_HALF_UP
        return int(Decimal(x).scaleb(-k).quantize(Decimal(1)))


def fit(v, p):
    return v if v is not None and -10 ** p < v < 10 ** p else None


def adjust(p, s):
    """DecimalType.adjustPrecisionScale with allowPrecisionLoss = true"""
    if p <= 38:
        return p, s
    return 38, max(38 - (p - s), min(s, 6))


def result_type(op, ta, tb):
    """Spark DecimalPrecision for (p, s) operands -> (p, s) of the result"""
    (p1, s1), (p2, s2) = ta, tb
    if op in ("add", "sub"):
        s = max(s1, s2)
        return adjust(max(p1 - s1, p2 - s2) + s + 1, s)
    if op == "mul":
        return adjust(p1 + p2 + 1, s1 + s2)
    s = max(6, s1 + p2 + 1)
    return adjust(p1 - s1 + s2 + s, s)


# the rules above at hand-checked points, so that a change to them is seen
RESULT_TYPES = {
    ("mul", (4, 2), (4, 1)): (9, 3), ("mul", (12, 2), (13, 2)): (26, 4), ("mul", (38, 10), (12, 2)): (38, 6),
    ("mul", (38, 20), (18, 10)): (38, 11), ("mul", (38, 22), (38, 22)): (38, 6), ("mul", (38, 30), (38, 30)): (38, 21),
    ("mul", (38, 0), (20, 0)): (38, 0), ("div", (12, 2), (12, 2)): (27, 15), ("div", (38, 6), (5, 0)): (38, 6),
    ("div", (1, 0), (1, 0)): (7, 6), ("div", (38, 0), (38, 32)): (38, 6), ("add", (38, 0), (38, 0)): (38, 0),
    ("add", (38, 2), (36, 6)): (38, 6), ("sub", (10, 2), (12, 5)): (14, 5), ("add", (38, 10), (38, 10)): (38, 9),
}


def unsupported(op, ta, tb):
    """the compiler raises B2Error: a divide that needs 10^k with k outside 0..38, an add/sub that loses scale"""
    rp, rs = result_type(op, ta, tb)
    if op == "div":
        k = rs - ta[1] + tb[1]
        return not 0 <= k <= 38
    if op in ("add", "sub"):
        return rs != max(ta[1], tb[1])
    return False


def ref_arith(op, a, b, ta, tb):
    if a is None or b is None:
        return None
    (_, s1), (_, s2) = ta, tb
    rp, rs = result_type(op, ta, tb)
    if op in ("add", "sub"):
        x, y = a * 10 ** (rs - s1), b * 10 ** (rs - s2)
        return fit(x + y if op == "add" else x - y, rp)
    if op == "mul":
        return fit(round_half_up(a * b, s1 + s2 - rs), rp)
    if b == 0:
        return None
    k = rs - s1 + s2
    with localcontext() as c:
        c.prec = 200
        c.rounding = ROUND_HALF_UP
        q = int((Decimal(a).scaleb(k) / Decimal(b)).quantize(Decimal(1)))
    return fit(q, rp)


def ref_cast(v, fs, tp, ts):
    """decimal (or integral, fs = 0) value v at scale fs -> DECIMAL(tp, ts)"""
    if v is None:
        return None
    return fit(v * 10 ** (ts - fs) if ts >= fs else round_half_up(v, fs - ts), tp)


def ref_cmp(op, a, b, sa, sb):
    if a is None or b is None:
        return (a is None and b is None) if op == "eqns" else None
    s = max(sa, sb)
    x, y = a * 10 ** (s - sa), b * 10 ** (s - sb)
    return {"eq": x == y, "eqns": x == y, "ne": x != y, "lt": x < y, "le": x <= y, "gt": x > y, "ge": x >= y}[op]


def ref_f64(v, s):
    return None if v is None else float(v) / float(10 ** s)


def ref_f32(v, s):
    return None if v is None else float(np.float32(ref_f64(v, s)))


# ---- data ------------------------------------------------------------------------------------------------------------
def digit_uniform(rnd, p, n):
    """d uniform in [0, p], value uniform in [10^(d-1), 10^d) (0 for d = 0), random sign"""
    out = []
    for _ in range(n):
        d = rnd.randint(0, p)
        v = 0 if d == 0 else rnd.randrange(10 ** (d - 1), 10 ** d)
        out.append(-v if rnd.random() < 0.5 else v)
    return out


def int_uniform(rnd, bits, n):
    lo, hi = -2 ** (bits - 1), 2 ** (bits - 1) - 1
    out = []
    for _ in range(n):
        d = rnd.randint(0, bits - 1)
        v = rnd.randrange(2 ** d) if d else 0
        out.append(max(lo, min(hi, -v if rnd.random() < 0.5 else v)))
    return out


def signs(x, y):
    return [(x, y), (-x, y), (x, -y), (-x, -y)]


def mul_low_digits(rnd, k, low, p1, p2, tries=400):
    """(x, y) with 0 < x < 10^p1, 0 < y < 10^p2 and x*y = low (mod 10^k): the product's last k digits are `low`"""
    m = 10 ** k
    for _ in range(tries):
        y = rnd.randrange(1, 10 ** rnd.randint(1, p2))
        if y % 2 == 0 or y % 5 == 0:
            continue
        x0 = low * pow(y, -1, m) % m
        if 0 < x0 < 10 ** p1:
            x = x0 + m * rnd.randint(0, (10 ** p1 - 1 - x0) // m)
            assert x * y % m == low
            return x, y
    return None


def mul_in_window(lo, hi, p1, p2, tries=3000):
    """(x, y) with lo <= x*y < hi, 0 < x < 10^p1, 0 < y < 10^p2, or None"""
    y = max(1, -(-lo // (10 ** p1 - 1)))
    for _ in range(tries):
        if y >= 10 ** p2:
            return None
        x = -(-lo // y)
        if x < 10 ** p1 and x * y < hi:
            return x, y
        y += 1
    return None


# ---- running -----------------------------------------------------------------------------------------------------------
def b2_column(b2, dt, scale, vals, with_nulls):
    valid = np.array([v is not None for v in vals], dtype=bool)
    ints = [0 if v is None else int(v) for v in vals]
    if dt == D128:
        data = np.array(ints, dtype=object)
    else:
        data = np.array(ints, dtype=NP_OF[dt])
    return b2.Column.from_numpy(data, dtype=dt, valid=valid if with_nulls else None, scale=scale)


def typ3(t):
    """(p, s) of a decimal, or an integral dtype code -> (dtype, p, s)"""
    return (t, 0, 0) if isinstance(t, int) else (dec_dtype(t[0]), t[0], t[1])


def fill_rows(rnd, types, edge_rows, n, nullable):
    """edge rows first, digit-uniform rows to n, then NULLs sprinkled over ~1/8 of the cells when nullable"""
    rows = [list(r) for r in edge_rows]
    while len(rows) < n:
        rows.append([int_uniform(rnd, INTS[t], 1)[0] if isinstance(t, int) else digit_uniform(rnd, t[0], 1)[0] for t in types])
    if nullable:
        for r in rows:
            for j in range(len(r)):
                if rnd.random() < 0.125:
                    r[j] = None
    return rows


def project_check(b2, types, rows, outputs, nullable):
    """outputs: [(Expr, expected (dtype, p, s), fn(row) -> value, kind)] with kind 'int', 'f64' or 'f32'"""
    cols = [b2_column(b2, typ3(t)[0], typ3(t)[2], [r[j] for r in rows], nullable) for j, t in enumerate(types)]
    out = b2.project(b2.Program([e for e, *_ in outputs]), b2.Table.from_columns(cols))
    assert out.num_rows == len(rows)
    for i, (e, etype, fn, kind) in enumerate(outputs):
        dt, p, s, _ = e.type()
        assert (dt, p, s) == etype, (i, e.sexpr, (dt, p, s), etype)
        got = out.column(i)
        assert (got.dtype, got.scale) == (etype[0], etype[2]), (i, e.sexpr)
        vals = got.to_pylist()
        for r, g in zip(rows, vals):
            want = fn(r)
            if kind != "int" and want is not None and g is not None:
                ok = struct.pack("<d", g) == struct.pack("<d", want)
            else:
                ok = g == want
            assert ok, "output %d %s row %r: got %r expected %r" % (i, e.sexpr, r, g, want)


def cols_of(b2, types, nullable):
    return [b2.col(j, *typ3(t), nullable=nullable) for j, t in enumerate(types)]


# ---- multiply ----------------------------------------------------------------------------------------------------------
def mul_instr(ta, tb):
    """the instruction and k that compile_arith picks for DECIMAL(ta) * DECIMAL(tb) columns"""
    mt = {D32: "I32", D64: "I64", D128: "I128"}
    p, s = ta[0] + tb[0] + 1, ta[1] + tb[1]
    rp, rs = adjust(p, s)
    ma, mb, rmt = mt[dec_dtype(ta[0])], mt[dec_dtype(tb[0])], mt[dec_dtype(rp)]
    if p <= 38:
        return ("V_MULW", 0) if rmt == "I128" and "I128" not in (ma, mb) else ("V_MUL " + rmt, 0)
    right = mb if ma == "I128" else ma     # the wide side goes left
    return ("V_MULDEC " + ("128" if right == "I128" else "64"), s - rs)


MUL_CASES = [  # (ta, tb, literal side or None)
    ((4, 2), (4, 1), None), ((9, 2), (8, 3), None), ((20, 2), (10, 2), None), ((12, 2), (13, 2), None),
    ((18, 4), (18, 4), None), ((38, 10), (12, 2), None), ((30, 10), (18, 9), None), ((38, 20), (18, 10), None),
    ((12, 2), (38, 10), None), ((38, 0), (20, 0), None), ((38, 10), (20, 5), None), ((38, 15), (30, 10), None),
    ((38, 16), (30, 10), None), ((38, 20), (38, 20), None), ((38, 22), (38, 22), None), ((38, 30), (38, 30), None),
    ((38, 38), (38, 7), None), ((38, 30), (38, 30), "left"), ((12, 2), (38, 10), "left"), ((38, 16), (30, 10), "right"),
]


def test_result_type_table():
    for (op, ta, tb), want in RESULT_TYPES.items():
        assert result_type(op, ta, tb) == want, (op, ta, tb)


def test_mul_instruction_coverage():
    reached = sorted({mul_instr(ta, tb) for ta, tb, _ in MUL_CASES})
    assert reached == [("V_MUL I128", 0), ("V_MUL I32", 0), ("V_MUL I64", 0),
                       ("V_MULDEC 128", 0), ("V_MULDEC 128", 9), ("V_MULDEC 128", 19), ("V_MULDEC 128", 20),
                       ("V_MULDEC 128", 34), ("V_MULDEC 128", 38), ("V_MULDEC 128", 39),
                       ("V_MULDEC 64", 6), ("V_MULDEC 64", 11), ("V_MULDEC 64", 19), ("V_MULW", 0)]


def mul_edge_rows(rnd, ta, tb):
    (p1, s1), (p2, s2) = ta, tb
    rp, rs = result_type("mul", ta, tb)
    k = s1 + s2 - rs
    big1, big2 = 10 ** p1 - 1, 10 ** p2 - 1
    rows = [(x, y) for x in (big1, -big1, 1, -1, 0) for y in (big2, -big2, 1, -1, 0)]
    if k > 0:
        half = 5 * 10 ** (k - 1)
        for low in (half, half - 1, half + 1, 10 ** k - 1, 1):
            for _ in range(3):
                xy = mul_low_digits(rnd, k, low, p1, p2)
                if xy:
                    rows += signs(*xy)
        if rp == 38:
            top = 10 ** (38 + k)
            for lo, hi in ((top - half, top + half),                 # rounds to exactly 10^38: NULL
                           ((10 ** 38 - 1) * 10 ** k, top - half),    # rounds to 10^38 - 1
                           (top - 10 ** k - half, top - 10 ** k)):    # rounds up to 10^38 - 1
                xy = mul_in_window(lo, hi, p1, p2)
                if xy:
                    rows += signs(*xy)
    for x, y in ((2 ** 64 + 3, 2 ** 64 + 5), (2 ** 127 // 10 ** 9, 10 ** 9 + 7), (10 ** 37 + 1, 10 ** 37 + 9)):
        if x <= big1 and y <= big2:
            rows += signs(x, y)
    return rows


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ta,tb,lit_side", MUL_CASES)
def test_multiply(b2, ta, tb, lit_side, nullable):
    rnd = random.Random(hash((ta, tb, lit_side, nullable)) & 0xffffffff)
    etype = typ3(result_type("mul", ta, tb))
    edge = mul_edge_rows(rnd, ta, tb)
    rows = fill_rows(rnd, [ta, tb], edge, N_FULL if not nullable else 3000, nullable)
    ca, cb = cols_of(b2, [ta, tb], nullable)
    if lit_side is None:
        outs = [(ca * cb, etype[:3], lambda r: ref_arith("mul", r[0], r[1], ta, tb), "int")]
    else:   # literals: every distinct operand of the edge rows on the literal side, a column on the other
        vals = sorted({r[0] if lit_side == "left" else r[1] for r in edge}, key=abs)
        vals = vals[:: max(1, len(vals) // 24)][:24]
        outs = []
        for v in vals:
            if lit_side == "left":
                e = b2.lit(v, *typ3(ta)) * cb
                outs.append((e, etype, lambda r, v=v: ref_arith("mul", v, r[1], ta, tb), "int"))
            else:
                e = ca * b2.lit(v, *typ3(tb))
                outs.append((e, etype, lambda r, v=v: ref_arith("mul", r[0], v, ta, tb), "int"))
    project_check(b2, [ta, tb], rows, outs, nullable)


# ---- divide ------------------------------------------------------------------------------------------------------------
# one type pair per k = rs - s1 + s2 in 0..38; results in DECIMAL32 (k 2..8), DECIMAL64 (9..17) and DECIMAL128
DIV_CASES = [((38, 6), (38, 0)), ((38, 5), (38, 0)), ((4, 4), (1, 0)), ((3, 3), (2, 0)), ((3, 2), (3, 0)),
             ((4, 1), (4, 0)), ((3, 0), (3, 0)), ((2, 0), (2, 1)), ((1, 0), (2, 2)), ((8, 0), (8, 0)),
             ((8, 0), (8, 1)), ((7, 0), (7, 3)), ((6, 0), (6, 5)), ((5, 0), (6, 6)), ((4, 0), (7, 6)),
             ((3, 0), (7, 7)), ((2, 0), (8, 7)), ((1, 0), (8, 8))] + [((38, 0), (38, 12 + j)) for j in range(21)]


def div_k(ta, tb):
    return result_type("div", ta, tb)[1] - ta[1] + tb[1]


def test_divide_k_coverage():
    assert [div_k(ta, tb) for ta, tb in DIV_CASES] == list(range(39))
    assert sorted({dec_dtype(result_type("div", ta, tb)[0]) for ta, tb in DIV_CASES}) == [D32, D64, D128]


def div_edge_rows(rnd, ta, tb):
    (p1, s1), (p2, s2) = ta, tb
    rp, rs = result_type("div", ta, tb)
    k = div_k(ta, tb)
    big1, big2 = 10 ** p1 - 1, 10 ** p2 - 1
    rows = [(x, y) for x in (big1, -big1, 1, -1, 0, 10 ** (p1 - 1)) for y in (1, -1, 2, -3, big2, -big2, 0)]
    # exact ties 2 * rem = |b|: b = 2^(k+1) d, a = d o (o odd) -> a 10^k / b = o 5^k / 2
    for _ in range(4):
        if 2 ** (k + 1) > big2:
            break
        d = rnd.randint(1, max(1, big2 // 2 ** (k + 1)))
        omax = min(big1 // d, 2 * 10 ** rp // 5 ** k)
        if omax < 1:
            break
        o = rnd.randrange(1, omax + 1) | 1
        if d * o <= big1:
            rows += signs(d * o, 2 ** (k + 1) * d)
            rows += signs(d * o - 1, 2 ** (k + 1) * d) if d * o > 1 else []
    # quotients of 10^38 - 1 and 10^38: a = ceil((T - 1/2) b / 10^k)
    if rp == 38:
        for t in (10 ** 38 - 1, 10 ** 38):
            for b in (10 ** k, 10 ** k + 1, big2, big2 // 3):
                if 0 < b <= big2:
                    a = -(-(2 * t - 1) * b // (2 * 10 ** k))
                    if a <= big1:
                        rows += signs(a, b)
    # the numerator |a| 10^k at or above 2^128 |b|
    if big1 * 10 ** k >= 2 ** 128:
        a = -(-(2 ** 128) // 10 ** k)
        rows += signs(a, 1) + signs(big1, 2)
    return rows


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ta,tb", DIV_CASES)
def test_divide(b2, ta, tb, nullable):
    rnd = random.Random(hash((ta, tb, nullable)) & 0xffffffff)
    rows = fill_rows(rnd, [ta, tb], div_edge_rows(rnd, ta, tb), N_FULL if not nullable else 2000, nullable)
    ca, cb = cols_of(b2, [ta, tb], nullable)
    etype = typ3(result_type("div", ta, tb))
    outs = [(ca / cb, etype, lambda r: ref_arith("div", r[0], r[1], ta, tb), "int")]
    if ta[0] <= 18:   # a literal numerator
        v = 10 ** ta[0] - 1
        outs.append((b2.lit(v, *typ3(ta)) / cb, etype, lambda r: ref_arith("div", v, r[1], ta, tb), "int"))
    project_check(b2, [ta, tb], rows, outs, nullable)


# ---- add / subtract ----------------------------------------------------------------------------------------------------
ADD_CASES = [((38, 0), (38, 0)), ((38, 6), (38, 6)), ((38, 2), (36, 6)), ((36, 6), (38, 2)), ((30, 0), (38, 6)),
             ((38, 4), (38, 6)), ((10, 2), (12, 5)), ((9, 0), (18, 3)), ((32, 0), (18, 6))]


def add_edge_rows(ta, tb):
    (p1, s1), (p2, s2) = ta, tb
    big1, big2 = 10 ** p1 - 1, 10 ** p2 - 1
    rows = [(x, y) for x in (big1, -big1, 1, -1, 0, 10 ** (p1 - 1)) for y in (big2, -big2, 1, -1, 0, 10 ** (p2 - 1))]
    rs = max(s1, s2)
    # around +-10^38 after rescaling, with the other side pulling back into range
    for c in (5, 9, 10, 15, 17, 18, 19, 20):
        for d in (0, 1, 4, 5, 9, 10):
            x, y = c * 10 ** (37 - (rs - s1)), d * 10 ** (37 - (rs - s2))
            for xx, yy in ((x, y - 1), (x - 1, y), (x + 1, y)):
                if abs(xx) <= big1 and abs(yy) <= big2:
                    rows += signs(xx, yy)
    return rows


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ta,tb", ADD_CASES)
def test_add_subtract(b2, ta, tb, nullable):
    rnd = random.Random(hash((ta, tb, nullable)) & 0xffffffff)
    rows = fill_rows(rnd, [ta, tb], add_edge_rows(ta, tb), N_FULL if not nullable else 2000, nullable)
    ca, cb = cols_of(b2, [ta, tb], nullable)
    ea, es = typ3(result_type("add", ta, tb)), typ3(result_type("sub", ta, tb))
    v = -(10 ** ta[0] - 1)
    outs = [(ca + cb, ea, lambda r: ref_arith("add", r[0], r[1], ta, tb), "int"),
            (ca - cb, es, lambda r: ref_arith("sub", r[0], r[1], ta, tb), "int"),
            (cb - ca, typ3(result_type("sub", tb, ta)), lambda r: ref_arith("sub", r[1], r[0], tb, ta), "int"),
            (b2.lit(v, *typ3(ta)) - cb, es, lambda r: ref_arith("sub", v, r[1], ta, tb), "int")]
    project_check(b2, [ta, tb], rows, outs, nullable)


# ---- casts ---------------------------------------------------------------------------------------------------------------
SRC = [(9, 4), (18, 6), (38, 10)]        # DECIMAL32, DECIMAL64, DECIMAL128
TGT_P = [9, 18, 30]                       # a DECIMAL32, DECIMAL64 and DECIMAL128 target
CAST_CASES = [(src, (tp, src[1] + d)) for src in SRC for tp in TGT_P for d in (2, 0, -2)] + [
    ((18, 0), (9, 2)), ((20, 0), (18, 0)), ((4, 3), (3, 2)), ((38, 0), (38, 18)), ((38, 20), (9, 0)), ((18, 2), (9, 9))]


def cast_edge_values(src, tgt):
    (fp, fs), (tp, ts) = src, tgt
    big = 10 ** fp - 1
    vals = [big, 1, 0, 10 ** (fp - 1)]
    ds = ts - fs
    if ds >= 0:
        c = -(-10 ** tp // 10 ** ds)
        vals += [c - 1, c]
    else:
        m = 10 ** -ds
        vals += [(10 ** tp - 1) * m + m // 2 - 1, (10 ** tp - 1) * m + m // 2, 10 ** tp * m]
    for bits in (32, 64):   # rescaled values that wrap to something small in a narrower machine type
        if ds >= 0:
            c = -(-2 ** bits // 10 ** ds)
            vals += [c, c + 1, 2 ** bits + 5]
        else:
            vals += [(2 ** bits + 5) * 10 ** -ds, (2 ** bits + 5) * 10 ** -ds + 10 ** -ds // 2]
    vals = sorted({v for v in vals if 0 <= v <= big})
    return vals + [-v for v in vals if v]


def test_cast_pair_coverage():
    pairs = {(dec_dtype(s[0]), dec_dtype(t[0]), (t[1] > s[1]) - (t[1] < s[1])) for s, t in CAST_CASES}
    assert len(pairs) == 27


def lit_outputs(b2, src_t3, src_scale, tgt, vals):
    """the same cast applied to literals (folded at compile time)"""
    etype = typ3(tgt)
    return [(b2.lit(v, *src_t3).cast(*etype), etype, lambda r, v=v: ref_cast(v, src_scale, *tgt), "int") for v in vals]


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("src,tgt", CAST_CASES)
def test_decimal_cast(b2, src, tgt, nullable):
    rnd = random.Random(hash((src, tgt, nullable)) & 0xffffffff)
    vals = cast_edge_values(src, tgt)
    rows = fill_rows(rnd, [src], [(v,) for v in vals], N_FULL if not nullable else 2000, nullable)
    (ca,) = cols_of(b2, [src], nullable)
    etype = typ3(tgt)
    outs = [(ca.cast(*etype), etype, lambda r: ref_cast(r[0], src[1], *tgt), "int")]
    project_check(b2, [src], rows, outs, nullable)
    if not nullable:
        for i in range(0, len(vals), 24):
            project_check(b2, [src], rows[:300], lit_outputs(b2, typ3(src), src[1], tgt, vals[i:i + 24]), False)


INT_CAST_CASES = [(it, (tp, s)) for it in INTS for tp in (9, 18, 38)
                  for s in sorted({0, 2, max(0, tp - len(str(2 ** (INTS[it] - 1))))})]


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("it,tgt", INT_CAST_CASES)
def test_integral_cast(b2, it, tgt, nullable):
    rnd = random.Random(hash((it, tgt, nullable)) & 0xffffffff)
    bits = INTS[it]
    lo, hi = -2 ** (bits - 1), 2 ** (bits - 1) - 1
    edge = {lo, hi, 0, 1, -1, lo + 1, hi - 1, 2 ** 32 + 5, -(2 ** 32 + 5), 42949673, -42949673}
    for e in (tgt[0] - tgt[1],):
        edge |= {10 ** e - 1, 10 ** e, -(10 ** e - 1), -10 ** e}
    vals = sorted(v for v in edge if lo <= v <= hi)
    rows = fill_rows(rnd, [it], [(v,) for v in vals], N_FULL if not nullable else 2000, nullable)
    (ca,) = cols_of(b2, [it], nullable)
    etype = typ3(tgt)
    outs = [(ca.cast(*etype), etype, lambda r: ref_cast(r[0], 0, *tgt), "int")]
    project_check(b2, [it], rows, outs, nullable)
    if not nullable:
        project_check(b2, [it], rows[:300], lit_outputs(b2, (it, 0, 0), 0, tgt, vals[:24]), False)


def test_literal_cast_range(b2):
    """a folded literal cast gives NULL exactly when the column cast does, including 10^30 -> DECIMAL(38,18)"""
    cases = [((38, 0), (38, 18), [10 ** 30, 10 ** 20 - 1, 10 ** 20, -10 ** 30, 2 ** 127 // 10 ** 9]),
             ((38, 0), (38, 10), [10 ** 28 - 1, 10 ** 28, 10 ** 37]), ((20, 0), (38, 18), [10 ** 20 - 1, 10 ** 19]),
             ((18, 0), (9, 2), [42949673, 9999999, 10 ** 7]), ((20, 0), (18, 0), [2 ** 64 + 5, 10 ** 18 - 1])]
    for src, tgt, vals in cases:
        rows = [(v,) for v in vals]
        (ca,) = cols_of(b2, [src], False)
        outs = [(ca.cast(*typ3(tgt)), typ3(tgt), lambda r: ref_cast(r[0], src[1], *tgt), "int")]
        outs += [(e, t, lambda r, f=f, row=row: f(row), k) for row, (e, t, f, k) in
                 zip(rows, lit_outputs(b2, typ3(src), src[1], tgt, vals))]
        project_check(b2, [src], rows, outs, False)
    assert ref_cast(10 ** 30, 0, 38, 18) is None


# ---- decimal -> float ----------------------------------------------------------------------------------------------------
FLOAT_TYPES = [(38, s) for s in range(39)] + [(9, s) for s in range(10)] + [(18, s) for s in range(19)]


@pytest.mark.parametrize("nullable", [False, True])
def test_decimal_to_float(b2, nullable):
    rnd = random.Random(17 + nullable)
    special = [2 ** 100 + 2 ** 47, 2 ** 100 + 2 ** 47 + 1, 2 ** 100 + 3 * 2 ** 47, 2 ** 53 + 1, 2 ** 63 - 1, 2 ** 64 + 2 ** 11,
               10 ** 38 - 1, 10 ** 18 - 1, 10 ** 9 - 1, 1, 5, 25]
    for i in range(0, len(FLOAT_TYPES), 12):
        types = FLOAT_TYPES[i:i + 12]
        edge = []
        for v in special:
            edge += [tuple(v if v < 10 ** t[0] else 1 for t in types), tuple(-v if v < 10 ** t[0] else -1 for t in types)]
        rows = fill_rows(rnd, types, edge, N_FULL if not nullable else 1000, nullable)
        cols = cols_of(b2, types, nullable)
        outs = []
        for j, (c, t) in enumerate(zip(cols, types)):
            outs.append((c.cast(O.FLOAT64), (O.FLOAT64, 0, 0), lambda r, j=j, s=t[1]: ref_f64(r[j], s), "f64"))
            outs.append((c.cast(O.FLOAT32), (O.FLOAT32, 0, 0), lambda r, j=j, s=t[1]: ref_f32(r[j], s), "f32"))
        project_check(b2, types, rows, outs, nullable)


# ---- comparisons ---------------------------------------------------------------------------------------------------------
CMP_CASES = [((10, 1), (12, 2)), ((5, 0), (20, 2)), ((38, 0), (38, 0)), ((9, 2), (18, 2)), ((37, 0), (38, 1)), ((3, 3), (30, 10))]
CMP_OPS = ["eq", "ne", "lt", "le", "gt", "ge", "eqns"]


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("ta,tb", CMP_CASES)
def test_compare(b2, ta, tb, nullable):
    rnd = random.Random(hash((ta, tb, nullable)) & 0xffffffff)
    (p1, s1), (p2, s2) = ta, tb
    m = min(s1, s2)
    umax = min((10 ** p1 - 1) // 10 ** (s1 - m), (10 ** p2 - 1) // 10 ** (s2 - m))
    edge = []
    for u in sorted({1, 7, umax, umax // 3, 10 ** (len(str(umax)) - 1)}):
        a, b = u * 10 ** (s1 - m), u * 10 ** (s2 - m)    # the same value u at scale m (1.0 vs 1.00)
        for d in (0, 1, -1):                              # and values one unit apart after rescaling
            if abs(b + d) < 10 ** p2:
                edge += [(a, b + d), (-a, -(b + d)), (a, -(b + d))]
    rows = fill_rows(rnd, [ta, tb], edge, N_FULL if not nullable else 2000, nullable)
    ca, cb = cols_of(b2, [ta, tb], nullable)
    ops = {"eq": ca == cb, "ne": ca != cb, "lt": ca < cb, "le": ca <= cb, "gt": ca > cb, "ge": ca >= cb,
           "eqns": ca.eq_null_safe(cb)}
    outs = [(ops[op], (O.BOOL8, 0, 0), lambda r, op=op: ref_cmp(op, r[0], r[1], s1, s2), "int") for op in CMP_OPS]
    project_check(b2, [ta, tb], rows, outs, nullable)


# ---- sweep over every DECIMAL(p, s) ------------------------------------------------------------------------------------
SWEEP_MUL_DIV = (38, 34)     # partner of a * b and a / b
SWEEP_ADD = (20, 4)          # partner of a + b
SWEEP_NARROW, SWEEP_WIDE = (7, 3), (38, 12)
SWEEP_TYPES = [(p, s) for p in range(1, 39) for s in range(p + 1)]


def test_sweep_every_precision_and_scale(b2):
    """a * b, a / b, a + b and two casts for every DECIMAL(p, s) a, three types per program"""
    assert len(SWEEP_TYPES) == 779
    rnd = random.Random(779)
    n = 64
    bmd = [1, -1, 0, 10 ** 38 - 1] + digit_uniform(rnd, SWEEP_MUL_DIV[0], n - 4)
    badd = digit_uniform(rnd, SWEEP_ADD[0], n)
    raised = {"div": 0, "add": 0}
    for group in range(0, len(SWEEP_TYPES), 3):
        idx = list(range(group, min(group + 3, len(SWEEP_TYPES))))
        # columns: the group's a columns, then the two partners
        cmd = b2.col(len(idx), D128, *SWEEP_MUL_DIV, nullable=False)
        cad = b2.col(len(idx) + 1, D128, *SWEEP_ADD, nullable=False)
        pending = []   # (type index, Expr, expected type, fn(a, b_muldiv, b_add))
        for c, j in enumerate(idx):
            t = SWEEP_TYPES[j]
            ca = b2.col(c, *typ3(t), nullable=False)
            for op, e, tb in (("mul", ca * cmd, SWEEP_MUL_DIV), ("div", ca / cmd, SWEEP_MUL_DIV), ("add", ca + cad, SWEEP_ADD)):
                if unsupported(op, t, tb):
                    with pytest.raises(b2.B2Error):
                        e.type()
                    raised[op] += 1
                    continue
                etype = typ3(result_type(op, t, tb))
                assert e.type()[:3] == etype, (op, t)
                pending.append((j, e, etype, lambda a, bm, ba, op=op, t=t, tb=tb: ref_arith(op, a, ba if op == "add" else bm, t, tb)))
            for tgt in (SWEEP_NARROW, SWEEP_WIDE):
                e = ca.cast(*typ3(tgt))
                assert e.type()[:3] == typ3(tgt)
                pending.append((j, e, typ3(tgt), lambda a, bm, ba, t=t, tgt=tgt: ref_cast(a, t[1], *tgt)))
        flush_group(b2, rnd, idx, pending, bmd, badd, n)
    # a / DECIMAL(38,34) needs 10^k with k = rs - s1 + 34 > 38 for 76 types (rs = 6 once adjusted, so s1 < 2);
    # a + DECIMAL(20,4) would lose scale (rs < s) for 168
    assert raised == {"div": 76, "add": 168}


def flush_group(b2, rnd, idx, pending, bmd, badd, n):
    avals = {}
    for j in idx:
        p, _ = SWEEP_TYPES[j]
        avals[j] = [10 ** p - 1, -(10 ** p - 1), 1, 0] + digit_uniform(rnd, p, n - 4)
    cols = [b2_column(b2, typ3(SWEEP_TYPES[j])[0], SWEEP_TYPES[j][1], avals[j], False) for j in idx]
    cols += [b2_column(b2, D128, SWEEP_MUL_DIV[1], bmd, False), b2_column(b2, D128, SWEEP_ADD[1], badd, False)]
    out = b2.project(b2.Program([e for _, e, _, _ in pending]), b2.Table.from_columns(cols))
    for i, (j, e, etype, fn) in enumerate(pending):
        got = out.column(i)
        assert (got.dtype, got.scale) == (etype[0], etype[2])
        g = got.to_pylist()
        for r in range(n):
            want = fn(avals[j][r], bmd[r], badd[r])
            assert g[r] == want, "%r %s row %d: a=%r b=%r got %r expected %r" % (
                SWEEP_TYPES[j], e.sexpr[0], r, avals[j][r], (bmd[r], badd[r]), g[r], want)
    pending.clear()


# ---- other VM hosts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nullable", [False, True])
def test_filter_on_overflowing_product(b2, nullable):
    """b2.filter (TMA-staged 16-byte columns) and b2.filter_row_ids keep a row only when a * b is not NULL and above
    the literal: the overflow-to-NULL of the 256-bit multiply decides rows"""
    ta, tb = (38, 10), (38, 10)
    rnd = random.Random(5 + nullable)
    rows = fill_rows(rnd, [ta, tb], mul_edge_rows(rnd, ta, tb), 3 * 65536 + 17, nullable)
    ca, cb = cols_of(b2, [ta, tb], nullable)
    rp, rs = result_type("mul", ta, tb)
    threshold = -10 ** 30
    pred = ca * cb > b2.lit(threshold, D128, rp, rs)
    keep = []
    for i, r in enumerate(rows):
        v = ref_arith("mul", r[0], r[1], ta, tb)
        if v is not None and v > threshold:
            keep.append(i)
    assert 0 < len(keep) < len(rows)
    cols = [b2_column(b2, D128, t[1], [r[j] for r in rows], nullable) for j, t in enumerate([ta, tb])]
    table = b2.Table.from_columns(cols)
    got = b2.filter(b2.Program([pred]), table).to_rows()
    assert got == [tuple(rows[i]) for i in keep]
    ids = b2.filter_row_ids(b2.Program([pred]), table).to_pylist()
    assert ids == keep
