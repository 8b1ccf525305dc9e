"""CPU-only: pins tests/vm_reference.py, the exact reference of the expression VM, two ways: against the oracle
(oracle.spark_cpu.eval_expr) on every operation both restate, and against answers Java gives."""
import math

import numpy as np
import pytest

from oracle import spark_cpu as O
from tests import vm_reference as R

INT_EDGES = {dt: [lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi]
             for dt, (lo, hi) in {R.INT8: (-2**7, 2**7 - 1), R.INT16: (-2**15, 2**15 - 1), R.INT32: (-2**31, 2**31 - 1),
                                  R.INT64: (-2**63, 2**63 - 1)}.items()}
FLOAT_EDGES = [math.nan, -math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, 2.2250738585072009e-308, 2.2250738585072014e-308,
               1.7976931348623157e308, 0.5, -0.5, 1.0, -1.0, 2.0**24 - 1, 2.0**24 + 1, 2147483647.0, 2147483647.5, 2.0**31,
               -2147483648.5, -2147483649.0, 2.0**63, -2.0**63, 300.7, -1e19, 1e19]


def _col(dt, vals, valid=None):
    with np.errstate(over="ignore"):
        v = np.array(vals, dtype=R.NP[dt])
    return O.OCol(v, np.ones(len(v), bool) if valid is None else np.asarray(valid, bool), (dt, 0, 0))


def _pairs(vals):
    return [a for a in vals for _ in vals], [b for _ in vals for b in vals]


def _assert_same(dt, got, exp):
    assert R.mismatches(dt, got[0], got[1], exp[0], exp[1]) == []


@pytest.mark.parametrize("dt", R.INT_TYPES + R.FLOAT_TYPES)
@pytest.mark.parametrize("op", ["add", "sub", "mul", "div", "mod", "pmod"])
def test_arith_matches_oracle(dt, op):
    vals = INT_EDGES[dt] if dt in INT_EDGES else FLOAT_EDGES
    xs, ys = _pairs(vals)
    a, b = _col(dt, xs), _col(dt, ys)
    exp = O.eval_expr((op, ("col", 0, a.typ), ("col", 1, b.typ)), [a, b])
    _assert_same(dt, R.arith(op, dt, a.values, b.values), (exp.values, exp.valid))


@pytest.mark.parametrize("dt", R.INT_TYPES + R.FLOAT_TYPES)
@pytest.mark.parametrize("op", ["eq", "ne", "lt", "le", "gt", "ge", "eqns"])
def test_compare_matches_oracle(dt, op):
    vals = INT_EDGES[dt] if dt in INT_EDGES else FLOAT_EDGES
    xs, ys = _pairs(vals)
    n = len(xs)
    va, vb = np.arange(n) % 5 != 0, np.arange(n) % 7 != 0
    a, b = _col(dt, xs, va), _col(dt, ys, vb)
    exp = O.eval_expr((op, ("col", 0, a.typ), ("col", 1, b.typ)), [a, b])
    _assert_same(R.BOOL8, R.compare(op, dt, a.values, b.values, va, vb), (exp.values, exp.valid))


@pytest.mark.parametrize("fdt", R.INT_TYPES + R.FLOAT_TYPES)
@pytest.mark.parametrize("tdt", (R.BOOL8,) + R.INT_TYPES + R.FLOAT_TYPES)
def test_numeric_casts_match_oracle(fdt, tdt):
    """the oracle casts int64 -> float32 through numpy, which rounds once too; every edge value agrees"""
    vals = INT_EDGES[fdt] + [2**24 + 1, 2**24 + 3] if fdt in INT_EDGES else FLOAT_EDGES
    vals = [v for v in vals if fdt not in INT_EDGES or INT_EDGES[fdt][0] <= v <= INT_EDGES[fdt][-1]]
    a = _col(fdt, vals)
    exp = O.eval_expr(("cast", ("col", 0, a.typ), (tdt, 0, 0)), [a])
    _assert_same(tdt, R.cast(fdt, tdt, a.values), (exp.values, exp.valid))


@pytest.mark.parametrize("case", [(R.DATE32, R.INT32), (R.DATE32, R.BOOL8), (R.DATE32, R.FLOAT64), (R.TIMESTAMP_US, R.INT64),
                                  (R.TIMESTAMP_US, R.INT8), (R.TIMESTAMP_US, R.FLOAT32), (R.TIMESTAMP_US, R.BOOL8),
                                  (R.INT32, R.TIMESTAMP_US), (R.INT64, R.TIMESTAMP_US), (R.BOOL8, R.TIMESTAMP_US)])
def test_datetime_casts_match_oracle(case):
    fdt, tdt = case
    vals = {R.DATE32: [-719162, -1, 0, 1, 2932896], R.TIMESTAMP_US: [-2**63, -1_000_001, -1_000_000, -999_999, -1, 0, 1, 10**6, 2**63 - 1],
            R.INT32: INT_EDGES[R.INT32], R.INT64: INT_EDGES[R.INT64] + [9223372036854, 9223372036855, -9223372036854, -9223372036855],
            R.BOOL8: [0, 1]}[fdt]
    a = _col(fdt, vals)
    exp = O.eval_expr(("cast", ("col", 0, a.typ), (tdt, 0, 0)), [a])
    _assert_same(tdt, R.cast(fdt, tdt, a.values), (exp.values, exp.valid))


def test_kleene_matches_oracle():
    tv = [(0, True), (1, True), (0, False)]
    xs, ys = _pairs(tv)
    x, vx = np.array([t[0] for t in xs], np.int8), np.array([t[1] for t in xs])
    y, vy = np.array([t[0] for t in ys], np.int8), np.array([t[1] for t in ys])
    a, b = O.OCol(x, vx, (R.BOOL8, 0, 0)), O.OCol(y, vy, (R.BOOL8, 0, 0))
    for op, fn in (("and", R.and_), ("or", R.or_)):
        exp = O.eval_expr((op, ("col", 0, a.typ), ("col", 1, b.typ)), [a, b])
        _assert_same(R.BOOL8, fn(x, vx, y, vy), (exp.values, exp.valid))
    exp = O.eval_expr(("not", ("col", 0, a.typ)), [a])
    _assert_same(R.BOOL8, R.not_(x, vx), (exp.values, exp.valid))


def test_year_matches_oracle():
    days = np.array([-719162, -1, 0, 59, 60, 365, 2932896], dtype=np.int32)
    exp = O.eval_expr(("year", ("col", 0, (R.DATE32, 0, 0))), [_col(R.DATE32, days)])
    _assert_same(R.INT32, R.year(days), (exp.values, exp.valid))


# ---- known Java answers -----------------------------------------------------------------------------------------------
def _one(fn, *args):
    vals, valid = fn(*args)
    return vals[0].item() if valid[0] else None


def test_java_integer_answers():
    MIN32, MIN64 = -2**31, -2**63
    a32 = lambda op, x, y: _one(R.arith, op, R.INT32, np.array([x], np.int32), np.array([y], np.int32))  # noqa: E731
    assert a32("div", MIN32, -1) == MIN32          # Integer.MIN_VALUE / -1
    assert a32("mod", MIN32, -1) == 0
    assert a32("pmod", MIN32, -1) == 0
    assert a32("div", -7, 2) == -3 and a32("mod", -7, 2) == -1 and a32("pmod", -7, 2) == 1
    assert a32("pmod", -1, MIN32) == 2**31 - 1     # (r + n) wraps to MAX_VALUE, MAX_VALUE % MIN_VALUE
    assert a32("pmod", MIN32, 3) == 1              # MIN % 3 = -2, -2 + 3 = 1
    assert a32("div", 5, 0) is None and a32("mod", 5, 0) is None and a32("pmod", 5, 0) is None
    assert a32("add", 2**31 - 1, 1) == MIN32 and a32("mul", 65536, 65536) == 0
    a8 = lambda op, x, y: _one(R.arith, op, R.INT8, np.array([x], np.int8), np.array([y], np.int8))  # noqa: E731
    assert a8("pmod", -128, 127) == 126            # byte pmod adds in int: -1 + 127 = 126, no wrap
    assert a8("div", -128, -1) == -128 and a8("mul", 16, 16) == 0
    a64 = lambda op, x, y: _one(R.arith, op, R.INT64, np.array([x], np.int64), np.array([y], np.int64))  # noqa: E731
    assert a64("div", MIN64, -1) == MIN64 and a64("mod", MIN64, -1) == 0
    assert _one(R.abs_, R.INT32, np.array([MIN32], np.int32)) == MIN32
    assert _one(R.neg, R.INT64, np.array([MIN64], np.int64)) == MIN64


def test_java_float_answers():
    f64 = lambda op, x, y: _one(R.arith, op, R.FLOAT64, np.array([x]), np.array([y]))  # noqa: E731
    assert f64("div", 1.0, -0.0) is None           # Spark: x / 0 is NULL, also for -0.0
    assert math.isnan(f64("mod", math.inf, 2.0)) and f64("mod", 5.0, math.inf) == 5.0
    assert math.copysign(1, f64("mod", -4.0, 2.0)) == -1    # -4.0 % 2.0 = -0.0 in Java
    assert f64("pmod", -1.0, 3.0) == 2.0 and f64("pmod", -7.5, -2.0) == -1.5
    assert f64("mod", 1e300, 3.0) == math.fmod(1e300, 3.0)  # exact, not x - trunc(x / y) * y
    a = _one(R.abs_, R.FLOAT64, np.array([-0.0]))
    assert a == 0.0 and math.copysign(1, a) == 1             # Math.abs(-0.0) = 0.0
    cmp = lambda op, x, y: _one(R.compare, op, R.FLOAT64, np.array([x]), np.array([y]))  # noqa: E731
    assert cmp("eq", math.nan, -math.nan) == 1 and cmp("gt", math.nan, math.inf) == 1 and cmp("eq", -0.0, 0.0) == 1


def test_java_cast_answers():
    c = lambda f, t, x: _one(R.cast, f, t, np.array([x], dtype=R.NP[f]))  # noqa: E731
    assert c(R.FLOAT32, R.INT8, 300.7) == 44                    # (byte)(int)300.7f
    assert c(R.FLOAT64, R.INT32, math.nan) == 0 and c(R.FLOAT32, R.INT64, math.nan) == 0
    assert c(R.FLOAT64, R.INT64, 1e19) == 2**63 - 1 and c(R.FLOAT64, R.INT64, -1e19) == -2**63
    assert c(R.FLOAT64, R.INT32, 2147483647.5) == 2**31 - 1 and c(R.FLOAT64, R.INT32, -2147483648.5) == -2**31
    assert c(R.FLOAT32, R.INT32, 2.0**31) == 2**31 - 1 and c(R.FLOAT64, R.INT16, 2.0**31) == -1   # (short)Integer.MAX_VALUE
    assert c(R.FLOAT64, R.INT32, -0.9) == 0 and c(R.FLOAT64, R.INT8, math.inf) == -1
    x = 2**54 + 2**30 + 1                                        # (float)x rounds once, to 2^54 + 2^31
    assert c(R.INT64, R.FLOAT32, x) == np.float32(2**54 + 2**31)
    assert np.float32(float(x)) == np.float32(2**54)            # the double rounding the reference must not do
    assert c(R.INT64, R.FLOAT32, 2**54 + 2**30 - 1) == np.float32(2**54)
    assert c(R.INT32, R.FLOAT32, 2**24 + 1) == np.float32(2**24) and c(R.INT32, R.FLOAT32, 2**24 + 3) == np.float32(2**24 + 4)
    assert c(R.INT64, R.FLOAT64, 2**53 + 1) == 2.0**53 and c(R.INT64, R.FLOAT64, 2**63 - 1) == 2.0**63
    assert c(R.FLOAT64, R.FLOAT32, 1e39) == np.float32(np.inf) and c(R.FLOAT64, R.FLOAT32, 1e-45) == np.float32(1e-45)
    assert c(R.FLOAT64, R.BOOL8, -0.0) == 0 and c(R.FLOAT64, R.BOOL8, math.nan) == 1


def test_java_datetime_answers():
    c = lambda f, t, x: _one(R.cast, f, t, np.array([x], dtype=R.NP[f]))  # noqa: E731
    assert c(R.TIMESTAMP_US, R.INT64, -1) == -1                 # floorDiv(-1 us, 10^6) = -1 s
    assert c(R.TIMESTAMP_US, R.INT64, -1_000_000) == -1 and c(R.TIMESTAMP_US, R.INT64, 999_999) == 0
    assert c(R.TIMESTAMP_US, R.INT32, -2**63) == R.wrap(-9223372036855, 32)
    assert c(R.TIMESTAMP_US, R.FLOAT64, 1_500_000) == 1.5 and c(R.TIMESTAMP_US, R.FLOAT64, -1) == -1e-6
    assert c(R.TIMESTAMP_US, R.BOOL8, 0) == 0 and c(R.TIMESTAMP_US, R.BOOL8, -5) == 1
    assert c(R.INT32, R.TIMESTAMP_US, -2**31) == -2**31 * 10**6 and c(R.BOOL8, R.TIMESTAMP_US, 1) == 1
    assert c(R.INT64, R.TIMESTAMP_US, 9223372036854) == 9223372036854000000
    assert c(R.INT64, R.TIMESTAMP_US, 9223372036855) == 2**63 - 1 and c(R.INT64, R.TIMESTAMP_US, -9223372036855) == -2**63
    for t in (R.BOOL8, R.INT8, R.INT32, R.INT64, R.FLOAT32, R.FLOAT64):
        assert c(R.DATE32, t, 18000) is None                     # date -> boolean / number is NULL
    for f, t in ((R.DATE32, R.TIMESTAMP_US), (R.TIMESTAMP_US, R.DATE32), (R.INT32, R.DATE32), (R.FLOAT64, R.TIMESTAMP_US)):
        with pytest.raises(ValueError):
            R.cast_one(f, t, 0)


def test_java_year_answers():
    y = lambda d: _one(R.year, np.array([d], np.int32))  # noqa: E731
    assert y(-719162) == 1 and y(-1) == 1969 and y(0) == 1970 and y(2932896) == 9999
    assert y(-719162 + 364) == 1 and y(-719162 + 365) == 2     # 0001 is not a leap year
    assert y(10957) == 2000 and y(10957 + 365) == 2000 and y(10957 + 366) == 2001   # 2000 is a leap year


def test_kleene_truth_tables():
    T, F, N = True, False, None
    assert [R.kleene_and(a, b) for a in (T, F, N) for b in (T, F, N)] == [T, F, N, F, F, F, N, F, N]
    assert [R.kleene_or(a, b) for a in (T, F, N) for b in (T, F, N)] == [T, T, T, T, F, N, T, N, N]
    x, v = np.array([1, 0, 1], np.int8), np.array([True, True, False])
    assert R.in_(R.INT32, np.array([1, 2, 3], np.int32), v, [1, None])[1].tolist() == [True, False, False]
    vals, valid = R.in_(R.INT32, np.array([1, 2], np.int32), np.array([True, True]), [1, 5])
    assert vals.tolist() == [1, 0] and valid.tolist() == [True, True]
    vals, valid = R.case_when(R.INT32, [(x, v, np.array([7, 8, 9], np.int32), np.ones(3, bool))])
    assert valid.tolist() == [True, False, False] and vals[0] == 7   # no ELSE: NULL when no branch is TRUE


def test_mismatch_rule():
    """any NaN matches any NaN; every other float must match bit for bit, so -0.0 is not 0.0"""
    f = np.array([np.nan, -0.0, 1.0])
    assert R.mismatches(R.FLOAT64, f, [True] * 3, np.array([-np.nan, -0.0, 1.0]), [True] * 3) == []
    assert [m[0] for m in R.mismatches(R.FLOAT64, f, [True] * 3, np.array([np.nan, 0.0, 1.0]), [True] * 3)] == [1]
    assert [m[0] for m in R.mismatches(R.INT32, np.array([0, 0]), [True, False], np.array([0, 0]), [False, False])] == [0]
