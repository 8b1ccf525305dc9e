"""The expression VM (vm.cuh, expr.cu) through every path it has, each case compared with tests/vm_reference.py.

 * Edge grids: every pair of integer edges {MIN, MIN+1, -2, -1, 0, 1, 2, MAX-1, MAX} of each width and of about 30 float
   edges (NaN of both signs and two payloads, +-inf, +-0.0, subnormals, the normal and finite limits, +-0.5, +-1, 2^24 +- 1,
   the int and long saturation bounds and their neighbours) through every binary operation, as column op column, column
   op literal, literal op column and literal op literal, again with NULLs over zero divisors and edge values, and against
   NULL literals.  Every value through the unary operations and every cast, including the rounding ties of int -> float
   and f64 -> f32 and the DATE32 / TIMESTAMP_US casts; every cast of a literal must equal the same cast of a column.
 * Loop paths: programs whose geometry (b2_program_info) puts K = 16, 5 to 7 and 1 to 3 rows on a thread under both register
   budgets, at 0, 1, 31, tile_rows +- 1 and 2 tile_rows - 1 rows, so the 8-row and 4-row batches, the remainder loop and
   the checked loop all run.
 * Host kernels: b2_project, b2_filter / b2_filter_row_ids / b2_filter_select below and above the TMA-staging threshold
   (with a 30-column predicate: 24 staged, 6 read from global memory) and with B2_FILTER_NO_TMA, b2_scan_aggregate with a
   predicate that drops the rows where a divisor is zero, and the high-cardinality group-by with and without a predicate
   and with B2_AGG_NO_FUSED_FIRST_PASS.  Each asserts from the kernel timings which kernel ran.
 * Register allocation: 64 instructions (65 is refused), 32 outputs, 64 input columns, 64 registers, deep trees whose
   destinations reuse source slots (the 1-byte pool that BOOL8 values and validity bytes share), outputs kept live while
   later outputs reuse slots, and V_ANDCMP conjunct fusion against the same predicate with one nullable term.
 * year() on every day from 0001-01-01 to 9999-12-31, and full three-valued truth tables of the Kleene operations."""
import datetime
import os

import numpy as np
import pytest

from tests import vm_reference as R

pytestmark = pytest.mark.gpu

BOOL8, INT8, INT16, INT32, INT64 = R.BOOL8, R.INT8, R.INT16, R.INT32, R.INT64
FLOAT32, FLOAT64, DATE32, TIMESTAMP_US = R.FLOAT32, R.FLOAT64, R.DATE32, R.TIMESTAMP_US
ERR_UNSUPPORTED = 5
VM_NT = 256

INT_EDGES = {dt: [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi]
             for dt, (lo, hi) in {INT8: (-2**7, 2**7 - 1), INT16: (-2**15, 2**15 - 1), INT32: (-2**31, 2**31 - 1),
                                  INT64: (-2**63, 2**63 - 1)}.items()}


def _f64_bits(*bits):
    return list(np.array(bits, dtype=np.uint64).view(np.float64))


def _f32_bits(*bits):
    return list(np.array(bits, dtype=np.uint32).view(np.float32))


_COMMON = [np.inf, -np.inf, 0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 2.0**24 - 1, 2.0**24 + 1, 2147483647.0, 2147483647.5, 2.0**31,
           -2147483648.5, -2147483649.0, 2.0**63, -2.0**63]
FLOAT_EDGES = {
    FLOAT64: np.array(_f64_bits(0x7ff8000000000000, 0xfff8000000000000, 0x7ff4000000000001, 0xfff000000000beef, 1, 0x000fffffffffffff,
                                0x0010000000000000, 0x7fefffffffffffff) + _COMMON +
                      [np.nextafter(2.0**63, 0), np.nextafter(2.0**63, np.inf), np.nextafter(-2.0**63, 0), np.nextafter(-2.0**63, -np.inf)],
                      dtype=np.float64),
    FLOAT32: np.array(_f32_bits(0x7fc00000, 0xffc00000, 0x7fa00001, 0xff80beef, 1, 0x007fffff, 0x00800000, 0x7f7fffff) +
                      [np.float32(v) for v in _COMMON] +
                      [np.nextafter(np.float32(2**63), np.float32(0)), np.nextafter(np.float32(2**63), np.float32(np.inf)),
                       np.nextafter(np.float32(-2**63), np.float32(0)), np.nextafter(np.float32(-2**63), np.float32(-np.inf))],
                      dtype=np.float32),
}
# values only cast, not paired: rounding ties and boundaries of the conversions
CAST_EXTRA = {
    INT32: [2**24 + 1, 2**24 + 3, -(2**24 + 1)],
    INT64: [2**54 + 2**30 - 1, 2**54 + 2**30 + 1, -(2**54 + 2**30 + 1), 2**53 + 1, 9223372036854, 9223372036855, -9223372036854,
            -9223372036855, -1_000_001, -1_000_000, -999_999, 999_999, 10**6, 1_500_000],
    FLOAT64: [1 + 2.0**-24, 1 + 3 * 2.0**-24, -(1 + 2.0**-24), 3.4028235677973366e38, 3.4028234663852886e38, 3.4028235677973362e38,
              1e-40, 1.5e-45, 7.006492321624085e-46, 7.006492321624087e-46, 1e39, -1e39, 300.7, -1e19, 1e19],
    FLOAT32: [300.7, -300.7, 127.9, 128.0, -129.0, 32767.5, 65535.0, 1e19, -1e19],
}
ALL_TYPES = (INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
NUMERIC_TARGETS = (BOOL8, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
ARITH = ("add", "sub", "mul", "div", "mod", "pmod")
CMP = ("eq", "ne", "lt", "le", "gt", "ge", "eqns")


def _edges(dt):
    return np.array(INT_EDGES[dt], dtype=R.NP[dt]) if dt in INT_EDGES else FLOAT_EDGES[dt]


def _cast_values(dt):
    base = list(_edges(dt)) if dt in ALL_TYPES else []
    if dt == BOOL8:
        base = [0, 1]
    if dt == DATE32:
        base = INT_EDGES[INT32] + [-719162, 0, 18000, 2932896]
    if dt == TIMESTAMP_US:
        base = INT_EDGES[INT64] + CAST_EXTRA[INT64]
    with np.errstate(over="ignore"):
        return np.array(base + CAST_EXTRA.get(dt, []) if dt != TIMESTAMP_US else base, dtype=R.NP[dt])


# ---- plumbing -------------------------------------------------------------------------------------------------------
def _column(b2, dt, vals, valid=None):
    return b2.Column.from_numpy(np.asarray(vals, dtype=R.NP[dt]), dtype=dt, valid=None if valid is None else np.asarray(valid, bool))


def _table(b2, cols):
    """cols: [(dtype, values, valid or None)]"""
    return b2.Table.from_columns([_column(b2, dt, v, ok) for dt, v, ok in cols])


def _lit(b2, v, dt):
    if v is None:
        return b2.lit(None, dt)
    if dt in (FLOAT32, FLOAT64):
        return b2.lit(float(v), dt)
    return b2.lit(int(v), dt)


def _run(b2, exprs, table, name="project_kernel"):
    """project `exprs` over `table` with kernel timing on -> ([(values, valid)], program info)"""
    prog = b2.Program(exprs)
    b2.profile_enable(True)
    try:
        out = b2.project(prog, table)
        ran = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    res = [out.column(i).to_numpy() for i in range(out.num_columns)]
    info = prog.info()
    if table.num_rows and name and info["ninstr"]:   # a program of plain columns and literals launches nothing
        assert name in ran, ran
    return res, info


def _check(dt, got, exp, what):
    bad = R.mismatches(dt, got[0], got[1], exp[0], exp[1])
    assert bad == [], "%s: (row, got, expected) %s" % (what, bad)


def _tile(exp, reps, n):
    return np.tile(exp[0], reps)[:n], np.tile(exp[1], reps)[:n]


def _bin(b2, op, a, b):
    return {"add": lambda: a + b, "sub": lambda: a - b, "mul": lambda: a * b, "div": lambda: a / b, "mod": lambda: a % b,
            "pmod": lambda: a.pmod(b), "eq": lambda: a == b, "ne": lambda: a != b, "lt": lambda: a < b, "le": lambda: a <= b,
            "gt": lambda: a > b, "ge": lambda: a >= b, "eqns": lambda: a.eq_null_safe(b)}[op]()


def _ref_bin(op, dt, x, y, vx=None, vy=None):
    if op in ARITH:
        return R.arith(op, dt, x, y, vx, vy)
    return R.compare(op, dt, x, y, vx, vy)


def _out_dt(op, dt):
    return dt if op in ARITH else BOOL8


# ---- edge grids -----------------------------------------------------------------------------------------------------
def _grid(dt):
    e = _edges(dt)
    g = len(e)
    return np.repeat(e, g), np.tile(e, g)


def _grid_validity(x, y):
    """NULLs over half of the zero divisors and over a spread of edge values on both sides"""
    i = np.arange(len(x))
    vy = ~(((y == 0) & (i % 2 == 0)) | (i % 7 == 3))
    vx = i % 5 != 1
    return vx, vy


@pytest.mark.parametrize("nullable", [False, True], ids=["plain", "nulls"])
@pytest.mark.parametrize("dt", ALL_TYPES)
def test_edge_grid_column_column(b2, dt, nullable):
    """every pair, repeated past two full tiles so that the fast loops run on the non-nullable outputs"""
    x, y = _grid(dt)
    g = len(x)
    vx, vy = _grid_validity(x, y) if nullable else (None, None)
    reps = -(-3 * 4096 // g) + 1
    n = g * reps - 5
    t = _table(b2, [(dt, np.tile(x, reps)[:n], None if vx is None else np.tile(vx, reps)[:n]),
                    (dt, np.tile(y, reps)[:n], None if vy is None else np.tile(vy, reps)[:n])])
    ca, cb = b2.col(0, dt, nullable=nullable), b2.col(1, dt, nullable=nullable)
    ops = ARITH + CMP
    got, info = _run(b2, [_bin(b2, op, ca, cb) for op in ops], t)
    assert n >= 2 * info["tile_rows"]
    for op, r in zip(ops, got):
        _check(_out_dt(op, dt), r, _tile(_ref_bin(op, dt, x, y, vx, vy), reps, n), "%s %s" % (op, R.NP[dt].__name__))


@pytest.mark.parametrize("side", ["column_literal", "literal_column"])
@pytest.mark.parametrize("dt", ALL_TYPES)
def test_edge_grid_literal(b2, dt, side):
    """column op literal and literal op column for every edge literal, NULL literals included; the column repeats the edges
    past two full tiles.  A non-zero literal divisor keeps the output non-nullable (and so on the fast loops)."""
    e = _edges(dt)
    g = len(e)
    reps = -(-3 * 4096 // g) + 1
    n = g * reps - 3
    t = _table(b2, [(dt, np.tile(e, reps)[:n], None)])
    c = b2.col(0, dt, nullable=False)
    ops = ARITH + CMP
    for v in list(e) + [None]:
        k = _lit(b2, v, dt)
        exprs = [_bin(b2, op, c, k) if side == "column_literal" else _bin(b2, op, k, c) for op in ops]
        got, _ = _run(b2, exprs, t)
        lv = np.full(g, 0 if v is None else v, dtype=R.NP[dt])
        lvalid = np.full(g, v is not None)
        for op, r in zip(ops, got):
            exp = _ref_bin(op, dt, e, lv, None, lvalid) if side == "column_literal" else _ref_bin(op, dt, lv, e, lvalid, None)
            _check(_out_dt(op, dt), r, _tile(exp, reps, n), "%s %s literal %r" % (op, side, v))
        if side == "column_literal" and v is not None and v != 0:   # a non-zero literal divisor cannot make a NULL
            assert not any(_bin(b2, op, c, k).type()[3] for op in ("div", "mod", "pmod"))


@pytest.mark.parametrize("dt", ALL_TYPES)
def test_edge_grid_literal_literal(b2, dt):
    """both sides literal: every pair, 32 outputs per program"""
    x, y = _grid(dt)
    t = _table(b2, [(INT32, np.arange(3, dtype=np.int32), None)])
    for op in ARITH + CMP:
        exp = _ref_bin(op, dt, x, y)
        for s in range(0, len(x), 32):
            got, _ = _run(b2, [_bin(b2, op, _lit(b2, a, dt), _lit(b2, b, dt)) for a, b in zip(x[s:s + 32], y[s:s + 32])], t)
            for j, r in enumerate(got):
                one = (np.repeat(exp[0][s + j], 3), np.repeat(exp[1][s + j], 3))
                _check(_out_dt(op, dt), r, one, "%s literal %r, %r" % (op, x[s + j], y[s + j]))


def _unary_exprs(b2, c, dt):
    """(label, expression, reference function of (values, valid)) for the unary operations and every numeric cast"""
    out = [("neg", -c, lambda v, ok: R.neg(dt, v, ok)), ("abs", c.abs(), lambda v, ok: R.abs_(dt, v, ok))]
    for to in NUMERIC_TARGETS + (TIMESTAMP_US,):
        if to == TIMESTAMP_US and dt in (FLOAT32, FLOAT64):
            continue
        out.append(("cast to %d" % to, c.cast(to), lambda v, ok, to=to: R.cast(dt, to, v, ok)))
    return out


@pytest.mark.parametrize("nullable", [False, True], ids=["plain", "nulls"])
@pytest.mark.parametrize("dt", ALL_TYPES)
def test_unary_and_casts_of_columns(b2, dt, nullable):
    v = _cast_values(dt)
    g = len(v)
    ok = (np.arange(g) % 3 != 1) if nullable else np.ones(g, bool)
    reps = -(-3 * 4096 // g) + 1
    n = g * reps - 7
    t = _table(b2, [(dt, np.tile(v, reps)[:n], np.tile(ok, reps)[:n] if nullable else None)])
    c = b2.col(0, dt, nullable=nullable)
    cases = _unary_exprs(b2, c, dt)
    got, _ = _run(b2, [e for _, e, _ in cases], t)
    for (label, e, ref), r in zip(cases, got):
        exp = ref(v, ok)
        _check(e.type()[0], r, _tile(exp, reps, n), "%s of %s" % (label, R.NP[dt].__name__))


def _cast_pairs():
    """(from, to) of every cast the VM compiles between the non-decimal types"""
    pairs = [(f, t) for f in ALL_TYPES + (BOOL8,) for t in NUMERIC_TARGETS if f != t]
    pairs += [(DATE32, t) for t in NUMERIC_TARGETS]
    pairs += [(TIMESTAMP_US, t) for t in NUMERIC_TARGETS]
    pairs += [(f, TIMESTAMP_US) for f in (BOOL8, INT8, INT16, INT32, INT64)]
    return pairs


@pytest.mark.parametrize("case", _cast_pairs(), ids=lambda c: "%d_to_%d" % c)
def test_cast_literal_folds_like_column(b2, case):
    """every value cast as a literal (folded at compile time or evaluated on literal operands) and as a column: both must be
    the reference.  An INT64 literal 2^54 + 2^30 + 1 cast to FLOAT32 is 2^54 + 2^31, not the 2^54 of a fold through double."""
    fdt, tdt = case
    v = _cast_values(fdt)
    ok = np.ones(len(v), bool)
    exp = R.cast(fdt, tdt, v, ok)
    t = _table(b2, [(fdt, v, None)])
    got, _ = _run(b2, [b2.col(0, fdt, nullable=False).cast(tdt)], t)
    _check(tdt, got[0], exp, "column cast %d -> %d" % case)
    for s in range(0, len(v), 8):
        got, _ = _run(b2, [_lit(b2, x, fdt).cast(tdt) for x in v[s:s + 8]], t, name=None)
        for j, r in enumerate(got):
            one = (np.repeat(exp[0][s + j], len(v)), np.repeat(exp[1][s + j], len(v)))
            _check(tdt, r, one, "literal %r cast %d -> %d" % ((v[s + j],) + case))
    got, _ = _run(b2, [b2.lit(None, fdt).cast(tdt)], t, name=None)
    assert not got[0][1].any()


def test_int64_literal_to_float32_rounds_once(b2):
    """the regression case of the literal fold: (float)(2^54 + 2^30 + 1) = 2^54 + 2^31 in Java, numpy and the VM's column path"""
    x = 2**54 + 2**30 + 1
    t = _table(b2, [(INT64, np.array([x]), None)])
    got, _ = _run(b2, [b2.lit(x, INT64).cast(FLOAT32), b2.col(0, INT64, nullable=False).cast(FLOAT32),
                       b2.lit(x, TIMESTAMP_US).cast(INT64).cast(FLOAT32)], t)
    assert got[0][0][0] == got[1][0][0] == np.float32(2**54 + 2**31)


def test_datetime_casts(b2):
    """GpuCast: date -> boolean / number is NULL, timestamp -> number is floorDiv seconds (or seconds in double), numbers ->
    timestamp are seconds (LONG saturating), booleans 0 / 1 microseconds"""
    ts = np.array([-1, -999_999, -1_000_000, -1_000_001, 0, 999_999, 1_500_000, -2**63, 2**63 - 1], dtype=np.int64)
    t = _table(b2, [(TIMESTAMP_US, ts, None), (DATE32, np.array([0, 1, -1, 18000, 2932896, -719162, 5, 6, 7], np.int32), None),
                    (INT64, np.array([9223372036854, 9223372036855, -9223372036854, -9223372036855, 0, 1, -1, 2**63 - 1, -2**63]), None)])
    c, d, s = b2.col(0, TIMESTAMP_US, nullable=False), b2.col(1, DATE32, nullable=False), b2.col(2, INT64, nullable=False)
    got, _ = _run(b2, [c.cast(INT64), c.cast(INT32), c.cast(FLOAT64), d.cast(INT32), d.cast(BOOL8), s.cast(TIMESTAMP_US)], t)
    assert got[0][0].tolist() == [-1, -1, -1, -2, 0, 0, 1, -9223372036855, 9223372036854]
    assert got[1][0].tolist()[:7] == [-1, -1, -1, -2, 0, 0, 1]
    assert got[2][0].tolist()[:7] == [-1e-6, -0.999999, -1.0, -1.000001, 0.0, 0.999999, 1.5]
    assert not got[3][1].any() and not got[4][1].any()
    assert got[5][0].tolist() == [9223372036854000000, 2**63 - 1, -9223372036854000000, -2**63, 0, 10**6, -10**6, 2**63 - 1, -2**63]
    for fdt, tdt in ((DATE32, TIMESTAMP_US), (TIMESTAMP_US, DATE32), (INT32, DATE32), (INT64, DATE32), (FLOAT64, TIMESTAMP_US),
                     (FLOAT32, TIMESTAMP_US), (BOOL8, DATE32)):
        with pytest.raises(b2.B2Error) as ei:
            b2.Program([b2.col(0, fdt).cast(tdt)])
        assert ei.value.code == ERR_UNSUPPORTED, (fdt, tdt)


# ---- loop paths -----------------------------------------------------------------------------------------------------
def _k_for(bpr):
    """rows per thread of a program with `bpr` register bytes per row (set_tile_geometry)"""
    budget = 72 * 1024 if bpr >= 24 else 40 * 1024
    return max(1, min(16, budget // (bpr * VM_NT))) if bpr > 0 else 16


def _program_at_k(b2, core, k, wide, c8, c64):
    """core plus INT64 and INT8 filler outputs (8 and 1 register bytes each, all kept live) until the program puts k rows on
    a thread under the wide (72 KB) or the narrow (40 KB) register budget -> (exprs, info), or None when core alone is
    already past that geometry"""
    exprs = [core]
    for _ in range(40):
        info = b2.Program(exprs).info()
        bpr, kk = info["bytes_per_row"], info["tile_rows"] // VM_NT
        if kk == k and (bpr >= 24) == wide:
            return exprs, info
        if len(exprs) == 32 or kk < k and (bpr >= 24 or not wide):
            return None
        if _k_for(bpr + 8) >= k and (wide or bpr + 8 < 24):
            exprs.append(c64 + b2.lit(len(exprs), INT64))
        else:
            exprs.append(c8 + b2.lit(len(exprs), INT8))
    return None


def _loop_data(n):
    """periodic columns (period 997, prime to every tile) so that the reference is computed on one period"""
    rng = np.random.default_rng(997)
    p = 997
    x = rng.integers(-2**31, 2**31, p, dtype=np.int64).astype(np.int32)
    y = rng.integers(-50, 50, p).astype(np.int32)
    x[:9] = INT_EDGES[INT32]
    y[:6] = [0, -1, 1, 0, -1, 2]
    vy = rng.random(p) > 0.2
    vy[0] = False   # a NULL over a zero divisor
    reps = -(-n // p) + 1
    return p, reps, x, y, vy


# (K, budget in KB): 8-row batches; 4-row batches + remainder under both budgets; remainder only (wide budget only: a narrow
# program always has K >= 6)
GEOMETRIES = [(16, 40), (7, 40), (6, 40), (7, 72), (5, 72), (3, 72), (2, 72), (1, 72)]


@pytest.mark.parametrize("k,budget", GEOMETRIES, ids=["K%d_%dKB" % g for g in GEOMETRIES])
def test_loop_paths(b2, k, budget):
    """each core expression in a program padded to the geometry, at 0, 1, 31, tile_rows - 1, tile_rows, tile_rows + 1 and
    2 tile_rows - 1 rows"""
    p, reps, x, y, vy = _loop_data(2 * 4096)
    cx, cy, cyn = b2.col(0, INT32, nullable=False), b2.col(1, INT32, nullable=False), b2.col(2, INT32, nullable=True)
    c8, c64 = b2.col(3, INT8, nullable=False), b2.col(4, INT64, nullable=False)
    three, seven, p3, p7, ones = b2.lit(3, INT32), b2.lit(7, INT32), np.full(p, 3, np.int32), np.full(p, 7, np.int32), np.ones(p, bool)
    and3 = R.and_(*R.and_(*R.compare("gt", INT32, x, p3), *R.compare("lt", INT32, y, p7)), *R.compare("ne", INT32, y, p3))
    cases = [   # (label, expression, dtype, reference over one period)
        ("column + literal", cx + three, INT32, R.arith("add", INT32, x, p3)),          # 8-row, 4-row and remainder loops
        ("column * column", cx * cy, INT32, R.arith("mul", INT32, x, y)),                # 4-row and remainder loops
        ("neg", -cx, INT32, R.neg(INT32, x)),                                            # unary fast loop
        ("column / 7", cx / seven, INT32, R.arith("div", INT32, x, p7)),                # non-nullable: fast loop
        ("column / nullable", cx / cyn, INT32, R.arith("div", INT32, x, y, ones, vy)),   # checked loop
        ("and of 3 comparisons", (cx > three) & (cy < seven) & (cy != three), BOOL8, and3),   # V_ANDCMP loops
        ("if, cast", b2.if_else(cy > three, cx, cy).cast(INT64), INT64,
         R.cast(INT32, INT64, *R.if_(INT32, *R.compare("gt", INT32, y, p3), x, ones, y, ones))),
        ("coalesce", cyn.coalesce(cx), INT32, R.coalesce(INT32, y, vy, x, ones)),
    ]
    ran = []
    for label, e, dt, ref in cases:
        built = _program_at_k(b2, e, k, budget == 72, c8, c64)
        if built is None:
            continue
        exprs, info = built
        assert info["tile_rows"] == k * VM_NT and (info["bytes_per_row"] >= 24) == (budget == 72), info
        ran.append(label)
        tr = info["tile_rows"]
        for n in sorted({0, 1, 31, tr - 1, tr, tr + 1, 2 * tr - 1}):
            r = max(reps, -(-n // p) + 1)
            t = _table(b2, [(INT32, np.tile(x, r)[:n], None), (INT32, np.tile(y, r)[:n], None),
                            (INT32, np.tile(y, r)[:n], np.tile(vy, r)[:n]), (INT8, np.zeros(n, np.int8), None),
                            (INT64, np.zeros(n, np.int64), None)])
            got, _ = _run(b2, exprs, t)
            _check(dt, got[0], _tile(ref, r, n), "%s, K=%d, %d rows" % (label, k, n))
    # only the widest core expression (13 register bytes per row) cannot reach K = 16
    assert len(ran) >= len(cases) - (1 if k == 16 else 0), ran


# ---- host kernels ---------------------------------------------------------------------------------------------------
def _ran(b2, fn):
    b2.profile_enable(True)
    try:
        res = fn()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return res, names


def _wide_filter_case(b2, n, seed):
    """30 INT32 columns; predicate ((c0 + ... + c29) * 3 - c0 / c1) % 7 < 4: the division by c1 == 0 is NULL, so are those
    rows' predicates (dropped)"""
    rng = np.random.default_rng(seed)
    cols = [rng.integers(-1000, 1000, n).astype(np.int32) for _ in range(30)]
    cols[1][rng.random(n) < 0.05] = 0
    s = np.sum(np.stack(cols).astype(np.int64), axis=0)
    q = np.where(cols[1] != 0, np.fix(cols[0] / np.where(cols[1] == 0, 1, cols[1])), 0).astype(np.int64)
    v = s * 3 - q
    keep = (cols[1] != 0) & (np.fmod(v, 7) < 4)
    exprs = [b2.col(i, INT32, nullable=False) for i in range(30)]
    acc = exprs[0]
    for e in exprs[1:]:
        acc = acc + e
    pred = ((acc * b2.lit(3, INT32) - exprs[0] / exprs[1]) % b2.lit(7, INT32)) < b2.lit(4, INT32)
    return cols, keep, pred


@pytest.mark.parametrize("n,tma", [(65_535, False), (65_536, True), (200_003, True), (200_003, False)],
                         ids=["below_threshold", "at_threshold", "staged", "no_tma"])
def test_filter_kernels(b2, n, tma):
    cols, keep, pred = _wide_filter_case(b2, n, n)
    t = b2.Table.from_columns([b2.Column.from_numpy(c) for c in cols])
    prog = b2.Program([pred])
    want = "filter_staged_kernel" if tma and n >= 65_536 else "filter_kernel"
    if not tma:
        os.environ["B2_FILTER_NO_TMA"] = "1"
    try:
        out, names = _ran(b2, lambda: b2.filter(prog, t))
        assert want in names and ({"filter_kernel", "filter_staged_kernel"} - {want}).isdisjoint(names), names
        for i in (0, 17, 29):
            assert np.array_equal(out.column(i).to_numpy()[0], cols[i][keep])
        ids, names = _ran(b2, lambda: b2.filter_row_ids(prog, t))
        assert want in names, names
        assert np.array_equal(ids.to_numpy()[0], np.flatnonzero(keep))
        sel, names = _ran(b2, lambda: b2.filter_select(prog, t, [29, 3]))
        assert want in names, names
        assert np.array_equal(sel.column(0).to_numpy()[0], cols[29][keep]) and np.array_equal(sel.column(1).to_numpy()[0], cols[3][keep])
    finally:
        os.environ.pop("B2_FILTER_NO_TMA", None)


@pytest.mark.parametrize("nkeys", [0, 1])
def test_scan_aggregate_with_predicate(b2, nkeys):
    """SUM / COUNT / MIN / MAX of y / (x % 3) under the predicate x % 3 != 0: every row the predicate drops divides by zero,
    and y / w divides by zero on some kept rows (NULL, so SUM skips it and COUNT does not count it)"""
    rng = np.random.default_rng(3 + nkeys)
    n = 100_003
    x = rng.integers(-10**6, 10**6, n).astype(np.int64)
    y = rng.integers(-10**9, 10**9, n).astype(np.int64)
    w = rng.integers(-3, 4, n).astype(np.int64)
    k = rng.integers(0, 37, n).astype(np.int32)
    t = b2.Table.from_columns([b2.Column.from_numpy(a) for a in (x, y, w, k)])
    cx, cy, cw, ck = (b2.col(i, dt, nullable=False) for i, dt in enumerate((INT64, INT64, INT64, INT32)))
    three = b2.lit(3, INT64)
    prog = b2.Program([cx % three != b2.lit(0, INT64), ck, cy / (cx % three), cy / cw])
    # key and aggregate columns count the outputs after the predicate
    aggs = [(b2.AGG_SUM, 1, INT64), (b2.AGG_COUNT, 1, INT64), (b2.AGG_MIN, 1, INT64), (b2.AGG_MAX, 1, INT64),
            (b2.AGG_SUM, 2, INT64), (b2.AGG_COUNT, 2, INT64), (b2.AGG_COUNT_ALL, 0, INT64)]
    out, names = _ran(b2, lambda: b2.scan_aggregate(prog, True, t, [0] if nkeys else [], aggs))
    assert names & {"aggregate_smem_kernel", "aggregate_global_kernel"}, names
    r = np.fmod(x, 3)
    kept = r != 0
    q1 = np.array([R._tdiv(int(a), int(b)) if b else 0 for a, b in zip(y, r)], dtype=np.int64)
    q2 = np.array([R._tdiv(int(a), int(b)) if b else 0 for a, b in zip(y, w)], dtype=np.int64)
    groups = k if nkeys else np.zeros(n, np.int32)
    rows = {}
    for g in np.unique(groups[kept]):
        m = kept & (groups == g)
        m2 = m & (w != 0)
        rows[int(g)] = [int(q1[m].sum()), int(m.sum()), int(q1[m].min()), int(q1[m].max()), int(q2[m2].sum()), int(m2.sum()), int(m.sum())]
    got = out.to_rows()
    if nkeys:
        got = {r[0]: list(r[1:]) for r in got}
    else:
        got = {0: list(got[0])}
    assert got == rows


A_MUL = 1_000_003


@pytest.mark.parametrize("mode", ["fused", "separate", "predicate"])
def test_radix_groupby_programs(b2, mode):
    """the high-cardinality group-by runs the VM in radix_rows_scatter_kernel (fixed 2048-row tiles, no predicate),
    radix_rows_kernel (B2_AGG_NO_FUSED_FIRST_PASS) or radix_rows_kernel with a predicate"""
    n, g = 1_300_007, 433_337
    rng = np.random.default_rng(11)
    key = (np.arange(n, dtype=np.int64) * A_MUL) % g
    v = rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)
    w = rng.integers(-10**6, 10**6, n, dtype=np.int64)
    t = b2.Table.from_columns([b2.Column.from_numpy(key), b2.Column.from_numpy(v), b2.Column.from_numpy(w)])
    ck, cv, cw = b2.col(0, INT64, nullable=False), b2.col(1, INT32, nullable=False), b2.col(2, INT64, nullable=False)
    val = cv.cast(INT64) * b2.lit(3, INT64) - cw / b2.lit(7, INT64)
    exprs = [ck, val, cv.abs().cast(INT64)]
    keep = np.ones(n, bool)
    if mode == "predicate":
        exprs = [(cw % b2.lit(5, INT64)) != b2.lit(0, INT64)] + exprs
        keep = np.fmod(w, 5) != 0
    prog = b2.Program(exprs)
    aggs = [(b2.AGG_SUM, 1, INT64), (b2.AGG_MAX, 2, INT64), (b2.AGG_COUNT_ALL, 0, INT64)]
    if mode == "separate":
        os.environ["B2_AGG_NO_FUSED_FIRST_PASS"] = "1"
    try:
        out, names = _ran(b2, lambda: b2.scan_aggregate(prog, mode == "predicate", t, [0], aggs))
    finally:
        os.environ.pop("B2_AGG_NO_FUSED_FIRST_PASS", None)
    want = "radix_rows_scatter_kernel" if mode == "fused" else "radix_rows_kernel"
    assert want in names and ({"radix_rows_scatter_kernel", "radix_rows_kernel"} - {want}).isdisjoint(names), names
    val_ref = v.astype(np.int64) * 3 - np.sign(w) * (np.abs(w) // 7)
    abs_ref = np.where(v == -2**31, -2**31, np.abs(v.astype(np.int64)))
    kk, vv, aa = key[keep], val_ref[keep], abs_ref[keep]
    order = np.argsort(kk, kind="stable")
    sk = kk[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    cols = [out.column(c).to_numpy()[0] for c in range(out.num_columns)]
    o = np.argsort(cols[0], kind="stable")
    assert np.array_equal(cols[0][o], sk[starts])
    assert np.array_equal(cols[1][o], np.add.reduceat(vv[order], starts))
    assert np.array_equal(cols[2][o], np.maximum.reduceat(aa[order], starts))
    assert np.array_equal(cols[3][o], np.diff(np.r_[starts, len(sk)]))


# ---- register allocation --------------------------------------------------------------------------------------------
def test_instruction_and_register_limits(b2):
    n = 5000
    x = np.arange(n, dtype=np.int64) - 2500
    t = _table(b2, [(INT64, x, None)])
    acc = b2.col(0, INT64, nullable=False)
    exp = [int(v) for v in x]
    for i in range(64):
        acc = acc + b2.lit(i, INT64) if i % 2 else acc * b2.lit(3, INT64)
        exp = [R.wrap(e + i if i % 2 else e * 3, 64) for e in exp]
    got, info = _run(b2, [acc], t)
    assert info["ninstr"] == 64 and info["nregs"] == 64, info
    assert got[0][0].tolist() == exp
    with pytest.raises(b2.B2Error) as ei:
        b2.Program([acc + b2.lit(1, INT64)])
    assert ei.value.code == ERR_UNSUPPORTED


def test_output_and_column_limits(b2):
    n = 300
    rng = np.random.default_rng(64)
    cols = [rng.integers(-100, 100, n).astype(np.int32) for _ in range(64)]
    t = b2.Table.from_columns([b2.Column.from_numpy(c) for c in cols])
    refs = [b2.col(i, INT32, nullable=False) for i in range(64)]
    acc = refs[0]
    for r in refs[1:]:
        acc = acc + r
    got, info = _run(b2, [acc], t)
    assert info["ninstr"] == 63 and info["nregs"] == 63, info
    assert got[0][0].tolist() == np.sum(np.stack(cols).astype(np.int64), axis=0).tolist()
    outs = [refs[i] * refs[63 - i] for i in range(32)]
    got, info = _run(b2, outs, t)
    assert info["ninstr"] == 32, info
    for i in range(32):
        assert np.array_equal(got[i][0], (cols[i].astype(np.int64) * cols[63 - i]).astype(np.int32))
    with pytest.raises(b2.B2Error):
        b2.Program(outs + [refs[0] + refs[1]])            # 33 outputs
    with pytest.raises(b2.B2Error):
        b2.Program([refs[0] + b2.col(64, INT32, nullable=False)])   # a 65th input column


def _random_tree(rng, b2, depth, kind, leaves):
    """random expression over nullable BOOL8 columns 0-2 and INT32 columns 3-5 -> (Expr, reference (values, valid), dtype)"""
    bcols, icols = leaves
    if depth == 0 or rng.random() < 0.15:
        if kind == "b":
            i = int(rng.integers(0, 3))
            return b2.col(i, BOOL8), bcols[i], BOOL8
        i = int(rng.integers(0, 3))
        return b2.col(3 + i, INT32), icols[i], INT32
    if kind == "b":
        op = rng.choice(["and", "or", "not", "if", "coalesce", "eqns", "lt", "isnull"])
        if op in ("and", "or"):
            (a, ra, _), (b, rb, _) = _random_tree(rng, b2, depth - 1, "b", leaves), _random_tree(rng, b2, depth - 1, "b", leaves)
            return (a & b if op == "and" else a | b), (R.and_ if op == "and" else R.or_)(*ra, *rb), BOOL8
        if op == "not":
            a, ra, _ = _random_tree(rng, b2, depth - 1, "b", leaves)
            return ~a, R.not_(*ra), BOOL8
        if op == "isnull":
            a, ra, _ = _random_tree(rng, b2, depth - 1, "i", leaves)
            return a.is_null(), (np.asarray(~ra[1], np.int8), np.ones(len(ra[1]), bool)), BOOL8
        if op in ("eqns", "lt"):
            (a, ra, _), (b, rb, _) = _random_tree(rng, b2, depth - 1, "i", leaves), _random_tree(rng, b2, depth - 1, "i", leaves)
            return (a.eq_null_safe(b) if op == "eqns" else a < b), R.compare(str(op), INT32, ra[0], rb[0], ra[1], rb[1]), BOOL8
    else:
        op = rng.choice(["if", "coalesce", "add", "div"])
        if op in ("add", "div"):
            (a, ra, _), (b, rb, _) = _random_tree(rng, b2, depth - 1, "i", leaves), _random_tree(rng, b2, depth - 1, "i", leaves)
            return (a + b if op == "add" else a / b), R.arith(str(op), INT32, ra[0], rb[0], ra[1], rb[1]), INT32
    dt = BOOL8 if kind == "b" else INT32
    if op == "if":
        p, rp, _ = _random_tree(rng, b2, depth - 1, "b", leaves)
        (a, ra, _), (b, rb, _) = _random_tree(rng, b2, depth - 1, kind, leaves), _random_tree(rng, b2, depth - 1, kind, leaves)
        return b2.if_else(p, a, b), R.if_(dt, *rp, *ra, *rb), dt
    (a, ra, _), (b, rb, _) = _random_tree(rng, b2, depth - 1, kind, leaves), _random_tree(rng, b2, depth - 1, kind, leaves)
    return a.coalesce(b), R.coalesce(dt, *ra, *rb), dt


@pytest.mark.parametrize("seed", range(12))
def test_deep_trees_reuse_slots(b2, seed):
    """2 to 4 outputs of random depth-6 trees over nullable booleans and ints: every destination may recycle a source slot,
    BOOL8 values and validity bytes share the 1-byte pool, and earlier outputs stay live while later ones reuse slots"""
    rng = np.random.default_rng(seed)
    n = 4096 * 2 + 77
    bvals = [(rng.integers(0, 2, n).astype(np.int8), rng.random(n) > 0.3) for _ in range(3)]
    ivals = [(rng.integers(-5, 6, n).astype(np.int32), rng.random(n) > 0.2) for _ in range(3)]
    t = _table(b2, [(BOOL8, v, ok) for v, ok in bvals] + [(INT32, v, ok) for v, ok in ivals])
    outs = []
    for _ in range(int(rng.integers(2, 5))):
        for _attempt in range(20):
            e, ref, dt = _random_tree(rng, b2, 6, rng.choice(["b", "i"]), (bvals, ivals))
            try:
                b2.Program([o[0] for o in outs] + [e])
            except b2.B2Error as err:   # more than 64 instructions or registers: draw another tree
                assert err.code == ERR_UNSUPPORTED
                continue
            outs.append((e, ref, dt))
            break
    got, info = _run(b2, [o[0] for o in outs], t)
    assert info["ninstr"] >= 8, info
    for j, ((e, ref, dt), r) in enumerate(zip(outs, got)):
        _check(dt, r, ref, "seed %d output %d" % (seed, j))


def test_andcmp_fusion_matches_unfused(b2):
    """(a > 1) AND (b < 5) AND (c != 3) fuses into V_ANDCMP when nothing is nullable; with c nullable it cannot, and both
    must equal the reference"""
    rng = np.random.default_rng(8)
    n = 3 * 4096 + 11
    a, b, c = (rng.integers(-3, 9, n).astype(np.int64) for _ in range(3))
    vc = rng.random(n) > 0.25
    t = _table(b2, [(INT64, a, None), (INT64, b, None), (INT64, c, None), (INT64, c, vc)])
    ca, cb = b2.col(0, INT64, nullable=False), b2.col(1, INT64, nullable=False)
    one, three, five = b2.lit(1, INT64), b2.lit(3, INT64), b2.lit(5, INT64)
    fused = (ca > one) & (cb < five) & (b2.col(2, INT64, nullable=False) != three)
    plain = (ca > one) & (cb < five) & (b2.col(3, INT64, nullable=True) != three)
    ones = np.ones(n, bool)
    ab = R.and_(*R.compare("gt", INT64, a, np.full(n, 1), ones, ones), *R.compare("lt", INT64, b, np.full(n, 5), ones, ones))
    got_f, info_f = _run(b2, [fused], t)
    got_p, info_p = _run(b2, [plain], t)
    assert info_f["ninstr"] < info_p["ninstr"], (info_f, info_p)
    _check(BOOL8, got_f[0], R.and_(*ab, *R.compare("ne", INT64, c, np.full(n, 3), ones, ones)), "fused")
    _check(BOOL8, got_p[0], R.and_(*ab, *R.compare("ne", INT64, c, np.full(n, 3), vc, ones)), "unfused")
    cnt = b2.filter_count(b2.Program([fused]), t)
    assert cnt == int(got_f[0][0].sum())


# ---- dates and logic ------------------------------------------------------------------------------------------------
def test_year_every_day(b2):
    """year() on each of the 3,652,059 days of 0001-01-01 .. 9999-12-31"""
    first = datetime.date(1, 1, 1).toordinal() - R.EPOCH_ORDINAL
    last = datetime.date(9999, 12, 31).toordinal() - R.EPOCH_ORDINAL
    days = np.arange(first, last + 1, dtype=np.int32)
    assert len(days) == 3_652_059
    lengths = [datetime.date(y + 1, 1, 1).toordinal() - datetime.date(y, 1, 1).toordinal() for y in range(1, 9999)] + [365]
    exp = np.repeat(np.arange(1, 10000, dtype=np.int32), lengths)
    t = _table(b2, [(DATE32, days, None)])
    got, _ = _run(b2, [b2.col(0, DATE32, nullable=False).year()], t)
    bad = np.flatnonzero(got[0][0] != exp)
    assert len(bad) == 0, [(int(days[i]), int(got[0][0][i]), int(exp[i])) for i in bad[:8]]


TV = [(1, True), (0, True), (0, False)]   # TRUE, FALSE, NULL


def test_kleene_truth_tables(b2):
    """AND, OR, NOT, <=>, IF and COALESCE over every combination of TRUE / FALSE / NULL as columns and as literals"""
    combos = [(p, q, r) for p in TV for q in TV for r in TV]
    cols = [(np.array([c[i][0] for c in combos], np.int8), np.array([c[i][1] for c in combos])) for i in range(3)]
    t = _table(b2, [(BOOL8, v, ok) for v, ok in cols])
    x, y, z = (b2.col(i, BOOL8) for i in range(3))
    (xv, xo), (yv, yo), (zv, zo) = cols
    n = len(combos)
    got, _ = _run(b2, [x & y, x | y, ~x, x.eq_null_safe(y), b2.if_else(x, y, z), x.coalesce(y), (x & y) | ~z], t)
    _check(BOOL8, got[0], R.and_(xv, xo, yv, yo), "and")
    _check(BOOL8, got[1], R.or_(xv, xo, yv, yo), "or")
    _check(BOOL8, got[2], R.not_(xv, xo), "not")
    _check(BOOL8, got[3], R.compare("eqns", BOOL8, xv, yv, xo, yo), "<=>")
    _check(BOOL8, got[4], R.if_(BOOL8, xv, xo, yv, yo, zv, zo), "if")
    _check(BOOL8, got[5], R.coalesce(BOOL8, xv, xo, yv, yo), "coalesce")
    _check(BOOL8, got[6], R.or_(*R.and_(xv, xo, yv, yo), *R.not_(zv, zo)), "(x and y) or not z")
    for lv, lo in TV:
        k = b2.lit(None if not lo else bool(lv), BOOL8)
        kv, ko = np.full(n, lv, np.int8), np.full(n, lo)
        got, _ = _run(b2, [x & k, k & x, x | k, k | x, x.eq_null_safe(k), k.eq_null_safe(x), b2.if_else(k, x, y), k.coalesce(x)], t)
        _check(BOOL8, got[0], R.and_(xv, xo, kv, ko), "and literal")
        _check(BOOL8, got[1], R.and_(kv, ko, xv, xo), "literal and")
        _check(BOOL8, got[2], R.or_(xv, xo, kv, ko), "or literal")
        _check(BOOL8, got[3], R.or_(kv, ko, xv, xo), "literal or")
        _check(BOOL8, got[4], R.compare("eqns", BOOL8, xv, kv, xo, ko), "<=> literal")
        _check(BOOL8, got[5], R.compare("eqns", BOOL8, kv, xv, ko, xo), "literal <=>")
        _check(BOOL8, got[6], R.if_(BOOL8, kv, ko, xv, xo, yv, yo), "if literal")
        _check(BOOL8, got[7], R.coalesce(BOOL8, kv, ko, xv, xo), "literal coalesce")


def test_case_when_and_in(b2):
    """CASE WHEN with and without ELSE over NULL conditions and NULL values; IN with and without a NULL in the list"""
    combos = [(p, q) for p in TV for q in TV]
    n = len(combos) * 3
    c1 = (np.array([c[0][0] for c in combos] * 3, np.int8), np.array([c[0][1] for c in combos] * 3))
    c2 = (np.array([c[1][0] for c in combos] * 3, np.int8), np.array([c[1][1] for c in combos] * 3))
    v = np.arange(n, dtype=np.int32) - 7
    vo = np.arange(n) % 4 != 2
    t = _table(b2, [(BOOL8, *c1), (BOOL8, *c2), (INT32, v, vo)])
    p, q, cv = b2.col(0, BOOL8), b2.col(1, BOOL8), b2.col(2, INT32)
    ten, twenty = b2.lit(10, INT32), b2.lit(20, INT32)
    ones = np.ones(n, bool)
    got, _ = _run(b2, [b2.case_when([(p, cv), (q, ten)]), b2.case_when([(p, ten), (q, cv)], twenty),
                       cv.isin([b2.lit(-7, INT32), b2.lit(3, INT32)]), cv.isin([b2.lit(-7, INT32), b2.lit(None, INT32)]),
                       cv.isin([])], t)
    _check(INT32, got[0], R.case_when(INT32, [(*c1, v, vo), (*c2, np.full(n, 10, np.int32), ones)]), "case without else")
    _check(INT32, got[1], R.case_when(INT32, [(*c1, np.full(n, 10, np.int32), ones), (*c2, v, vo)], (np.full(n, 20, np.int32), ones)),
           "case with else")
    _check(BOOL8, got[2], R.in_(INT32, v, vo, [-7, 3]), "in")
    _check(BOOL8, got[3], R.in_(INT32, v, vo, [-7, None]), "in with NULL")
    _check(BOOL8, got[4], R.in_(INT32, v, vo, []), "in ()")
