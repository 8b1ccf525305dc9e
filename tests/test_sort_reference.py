"""CPU tests (no GPU): the rank-based sort reference (tests/sort_reference.py) agrees with the comparator oracle
(oracle.spark_relational.sort_order) on small random tables of every type, direction and null placement, and with
hand-written answers at the edges of Spark's order."""
import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from tests import datagen as G
from tests import sort_reference as S

TYPES = [(O.BOOL8, 0, 0), (O.INT8, 0, 0), (O.INT16, 0, 0), (O.INT32, 0, 0), (O.INT64, 0, 0), (O.FLOAT32, 0, 0), (O.FLOAT64, 0, 0),
         (O.DATE32, 0, 0), (O.TIMESTAMP_US, 0, 0), (O.DECIMAL32, 9, 2), (O.DECIMAL64, 18, 4), (O.DECIMAL128, 38, 6), (O.STRING, 0, 0)]
ORDERS = [(1, 1), (1, 0), (0, 1), (0, 0)]


def col(values, typ, valid=None):
    values = np.array(values, dtype=object) if typ[0] in (O.STRING, O.DECIMAL128, O.DECIMAL64, O.DECIMAL32) else np.asarray(values)
    return O.OCol(values, np.ones(len(values), bool) if valid is None else np.asarray(valid, bool), typ)


def random_col(rng, typ, n):
    if typ[0] == O.TIMESTAMP_US:
        c = G.gen_column(rng, (O.INT64, 0, 0), n, null_frac=0.2)
        c = O.OCol(c.values, c.valid, typ)
    else:
        c = G.gen_column(rng, typ, n, null_frac=0.2, distinct=None if typ[0] == O.BOOL8 else 12)
    if typ[0] in S.FLOATS:
        c.values[rng.choice(n, 6, replace=False)] = [np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf]
        c.values[rng.choice(n, 6, replace=False)] *= -1
    elif typ[0] == O.STRING:
        extra = [b"", b"a\0", b"\x80", b"\xff", b"\x7f", "été".encode()]
        c.values[rng.choice(n, len(extra), replace=False)] = extra
    elif typ[0] not in (O.BOOL8,):
        neg = rng.random(n) < 0.5
        if O.is_decimal(typ[0]):
            c.values = np.array([-v if s else v for v, s in zip(c.values, neg)], dtype=object)
        else:
            c.values = np.where(neg, -c.values, c.values).astype(c.values.dtype)
    return c


@pytest.mark.parametrize("typ", TYPES)
@pytest.mark.parametrize("asc,nf", ORDERS)
def test_reference_matches_comparator_oracle(typ, asc, nf):
    rng = np.random.default_rng(typ[0] * 8 + asc * 2 + nf)
    n = 300
    c = random_col(rng, typ, n)
    assert S.sort_order([c], [(0, asc, nf)]).tolist() == R.sort_order([c], [(0, asc, nf)])


@pytest.mark.parametrize("seed", range(6))
def test_reference_matches_comparator_oracle_multi_key(seed):
    rng = np.random.default_rng(100 + seed)
    n = 400
    types = [TYPES[i] for i in rng.choice(len(TYPES), 3, replace=False)]
    cols = [random_col(rng, t, n) for t in types]
    keys = [(k, int(rng.integers(0, 2)), int(rng.integers(0, 2))) for k in range(3)]
    assert S.sort_order(cols, keys).tolist() == R.sort_order(cols, keys)
    # merge of sorted pieces = stable order of their concatenation; top-N = its prefix
    parts = [[O.OCol(c.values[a:b], c.valid[a:b], c.typ) for c in cols] for a, b in ((0, 150), (150, 150), (150, 400))]
    parts = [[O.OCol(c.values[S.sort_order(p, keys)], c.valid[S.sort_order(p, keys)], c.typ) for c in p] for p in parts]
    cat = S.concat(parts)
    assert S.merge(parts, keys).tolist() == R.sort_order(cat, keys)
    assert S.top_n(cols, keys, 17).tolist() == R.sort_order(cols, keys)[:17]


def _pair(x, y, i, j):
    """the two-row table [x[i], y[j]]"""
    vals = np.empty(2, dtype=x.values.dtype)
    vals[0], vals[1] = x.values[i], y.values[j]
    return [O.OCol(vals, np.array([x.valid[i], y.valid[j]]), x.typ)]


@pytest.mark.parametrize("typ", [t for t in TYPES if t[0] != O.STRING])
@pytest.mark.parametrize("asc,nf", ORDERS)
def test_bounds_count_rows_before_the_probe(typ, asc, nf):
    """lower = the sorted rows that sort strictly before the probe row, upper = those that do not sort after it, with
    "before" taken from the comparator oracle"""
    rng = np.random.default_rng(typ[0] * 8 + asc * 2 + nf + 1000)
    s, p = random_col(rng, typ, 60), random_col(rng, typ, 30)
    keys = [(0, asc, nf)]
    perm = S.sort_order([s], keys)
    s = O.OCol(s.values[perm], s.valid[perm], s.typ)
    lo, hi = np.zeros(30, np.int64), np.zeros(30, np.int64)
    for i in range(30):
        for j in range(60):
            s_first = R.sort_order(_pair(p, s, i, j), keys) == [1, 0]   # s[j] sorts strictly before p[i]
            p_first = R.sort_order(_pair(s, p, j, i), keys) == [1, 0]   # p[i] sorts strictly before s[j]
            lo[i] += s_first
            hi[i] += not p_first
    assert S.bounds([s], [p], keys, False).tolist() == lo.tolist()
    assert S.bounds([s], [p], keys, True).tolist() == hi.tolist()


def _order(values, typ, asc=1, nf=1, valid=None):
    return S.sort_order([col(values, typ, valid)], [(0, asc, nf)]).tolist()


def test_nan_sorts_after_infinity_and_all_nans_tie():
    nan_neg = -np.float64(np.nan)
    vals = [np.nan, np.inf, 1.0, nan_neg, -np.inf]
    assert _order(vals, (O.FLOAT64, 0, 0)) == [4, 2, 1, 0, 3]
    assert _order(vals, (O.FLOAT64, 0, 0), asc=0) == [0, 3, 1, 2, 4]
    f32 = np.array([0x7fc00000, 0x7f800000, 0xffc00001, 0x7f800001], np.uint32).view(np.float32)   # NaN, +inf, -NaN, sNaN
    assert _order(f32, (O.FLOAT32, 0, 0)) == [1, 0, 2, 3]


def test_negative_zero_ties_with_zero_in_input_order():
    assert _order([0.0, -0.0, 0.0, -0.0, -1e-300], (O.FLOAT64, 0, 0)) == [4, 0, 1, 2, 3]
    assert _order([-0.0, 0.0, 5e-324], (O.FLOAT64, 0, 0), asc=0) == [2, 0, 1]


def test_strings_compare_by_unsigned_bytes_then_length():
    vals = [b"ab", b"a\0\0", b"a", b"a\0", b"\x80", b"\x7f", b"", b"\xff"]
    got = [vals[i] for i in _order(vals, (O.STRING, 0, 0))]
    assert got == [b"", b"a", b"a\0", b"a\0\0", b"ab", b"\x7f", b"\x80", b"\xff"]
    got = [vals[i] for i in _order(vals, (O.STRING, 0, 0), asc=0)]
    assert got == [b"\xff", b"\x80", b"\x7f", b"ab", b"a\0\0", b"a\0", b"a", b""]


def test_null_placement_does_not_follow_direction():
    vals, valid = [3, 0, 1, 0, 2], [True, False, True, False, True]
    t = (O.INT32, 0, 0)
    assert _order(vals, t, 1, 1, valid) == [1, 3, 2, 4, 0]
    assert _order(vals, t, 1, 0, valid) == [2, 4, 0, 1, 3]
    assert _order(vals, t, 0, 1, valid) == [1, 3, 0, 4, 2]
    assert _order(vals, t, 0, 0, valid) == [0, 4, 2, 1, 3]


def test_long_min_first_under_asc():
    vals = np.array([0, 2**63 - 1, -1, -2**63, 1, -2**63 + 1], np.int64)
    assert _order(vals, (O.INT64, 0, 0)) == [3, 5, 2, 0, 4, 1]
    assert _order(vals, (O.TIMESTAMP_US, 0, 0), asc=0) == [1, 4, 0, 2, 5, 3]


def test_decimal128_orders_as_integers():
    vals = [-(10**38 - 1), 2**64, -1, 0, 2**64 - 1, -2**64, 10**38 - 1, -2**63]
    got = [vals[i] for i in _order(vals, (O.DECIMAL128, 38, 0))]
    assert got == sorted(vals)


def test_bounds_hand_written():
    s = col([1, 3, 3, 5], (O.INT32, 0, 0))
    p = col([0, 3, 4, 9, 0], (O.INT32, 0, 0), [True, True, True, True, False])
    assert S.bounds([s], [p], [(0, 1, 1)], False).tolist() == [0, 1, 3, 4, 0]
    assert S.bounds([s], [p], [(0, 1, 1)], True).tolist() == [0, 3, 3, 4, 0]
    assert S.bounds([s], [p], [(0, 1, 0)], False).tolist() == [0, 1, 3, 4, 4]
    sd = col([5, 3, 3, 1], (O.INT32, 0, 0))
    assert S.bounds([sd], [p], [(0, 0, 0)], False).tolist() == [4, 1, 1, 0, 4]
    assert S.bounds([sd], [p], [(0, 0, 0)], True).tolist() == [4, 3, 1, 0, 4]
    z = col([-1.0, -0.0, 0.0, np.nan], (O.FLOAT64, 0, 0))
    q = col([0.0, -0.0, np.nan, np.inf], (O.FLOAT64, 0, 0))
    assert S.bounds([z], [q], [(0, 1, 1)], False).tolist() == [1, 1, 3, 3]
    assert S.bounds([z], [q], [(0, 1, 1)], True).tolist() == [3, 3, 4, 3]
    e = col(np.zeros(0, np.int32), (O.INT32, 0, 0))
    assert S.bounds([e], [p], [(0, 1, 1)], True).tolist() == [0] * 5


def test_merge_keeps_ties_in_table_order():
    a = [col([1, 2, 2], (O.INT64, 0, 0)), col([0, 1, 2], (O.INT64, 0, 0))]
    b = [col([2, 2], (O.INT64, 0, 0)), col([10, 11], (O.INT64, 0, 0))]
    e = [col(np.zeros(0, np.int64), (O.INT64, 0, 0)), col(np.zeros(0, np.int64), (O.INT64, 0, 0))]
    assert S.merge([a, e, b], [(0, 1, 1)]).tolist() == [0, 1, 2, 3, 4]
    assert S.merge([b, a], [(0, 1, 1)]).tolist() == [2, 0, 1, 3, 4]
    assert S.top_n(a, [(0, 0, 0)], 2).tolist() == [1, 2]
    assert S.top_n(a, [(0, 0, 0)], 0).tolist() == []
    assert S.top_n(a, [(0, 0, 0)], 10).tolist() == [1, 2, 0]
