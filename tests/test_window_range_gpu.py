"""RANGE frames with value offsets on the GPU (B2_FRAME_RANGE_VALUE through b2_window and GpuWindowExec) against the row-at-a-time
oracle (tests/window_range_oracle.py): exact, floats bit for bit (any NaN matches any NaN; the float inputs are integers, +-inf and
NaN, so every partial sum is exact in double whatever the association)."""
import math

import numpy as np
import pytest

from oracle import spark_window as W
from tests import window_range_oracle as R
from tests.test_window_gpu import _batches, _column, _kernels, _same

pytestmark = pytest.mark.gpu

TILE = 1024   # rows per tile of the range-query structure (window.cu WIN_TILE)
INVALID, UNSUPPORTED = 1, 5
BIG64 = 2 ** 63 - 2
ORDER_POOLS = {   # few distinct values per type, so peer groups form, with the type's edges
    "INT8": ([-128, 127, -1, 0, 1, 3, 100, -100], [127, 300]),
    "INT16": ([-32768, 32767, 0, 2, 5, -5, 1000], [3, 70000]),
    "INT32": ([-2 ** 31, 2 ** 31 - 1, 0, 1, 4, -9, 10 ** 6], [2, 2 ** 32]),
    "INT64": ([-2 ** 63, -2 ** 63 + 2, 2 ** 63 - 1, 2 ** 63 - 3, 0, 1, -1, 7], [3, BIG64]),
    "DATE32": ([0, 1, 7, 8, 30, -365, 20000], [7, 2 ** 40]),
    "TIMESTAMP_US": ([0, 10 ** 6, 86400 * 10 ** 6, 86400 * 10 ** 6 + 1, -5, 2 ** 62], [10 ** 6, 86400 * 10 ** 6]),
    "DECIMAL32": ([-(10 ** 9 - 1), 10 ** 9 - 1, 0, 150, 250, -100], [100, BIG64]),
    "DECIMAL64": ([-(10 ** 18 - 1), 10 ** 18 - 1, 0, 12345, 12346, -7], [1, 10 ** 18]),
    "DECIMAL128": ([-(10 ** 38 - 1), 10 ** 38 - 1, 0, 10 ** 30, 10 ** 30 + 2, -3], [2, BIG64]),
}


def _same_rows(a, b):
    """two lists of column lists, floats bit for bit with any NaN matching any NaN"""
    return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))


def _frames(ks):
    out = [(1, 3), (-3, -1), (0, 0), (0, None)]
    for k in ks:
        out += [(-k, 0), (-k, k), (0, k), (None, k), (-k, None)]
    return out


def _value_cols(m, rng, n, nullable):
    f = [float(x) for x in rng.integers(-1000, 1000, n)]
    for j in rng.integers(0, max(n, 1), n // 50 + 1) if n else []:
        f[int(j)] = [math.inf, -math.inf, math.nan][int(j) % 3]
    i64 = [int(x) for x in rng.integers(-2 ** 62, 2 ** 62, n)]
    d18 = [int(x) for x in rng.integers(-10 ** 17, 10 ** 17, n)]
    if nullable:
        f, i64, d18 = ([None if rng.random() < 0.1 else v for v in c] for c in (f, i64, d18))
    return {"i64": i64, "f64": f, "d18": d18}


def _funcs(m, frame, c):
    """(WindowFunc, oracle kind, value column, vtype) for one frame; c = the first value column's index"""
    lo, up = frame
    fr = m.range_between(lo, up)
    return [(m.win_sum(c, fr), W.SUM, "i64", "int"), (m.win_sum(c + 1, fr), W.SUM, "f64", "float"),
            (m.win_sum(c + 2, fr, m.DECIMAL128, 28), W.SUM, "d18", "decimal"), (m.win_count(c + 1, fr), W.COUNT, "f64", "int"),
            (m.win_count_all(fr), W.COUNT_ALL, None, "int"), (m.win_min(c, fr), W.MIN, "i64", "int"), (m.win_max(c + 1, fr), W.MAX, "f64", "float"),
            (m.win_min(c + 1, fr), W.MIN, "f64", "float")]


def _sorted_table(m, rng, n, nparts, otype, order_vals, asc, nulls_first, nullable):
    """(table sorted on the GPU by (p, o), its columns as Python lists); columns: p INT32, o, i64, f64, d18"""
    dt = getattr(m, otype)
    o = [order_vals[int(i)] for i in rng.integers(0, len(order_vals), n)]
    if nullable:
        o = [None if rng.random() < 0.15 else v for v in o]
    p = [int(x) for x in rng.integers(0, max(nparts, 1), n)]
    vals = _value_cols(m, rng, n, nullable)
    scale = 2 if otype.startswith("DECIMAL") else 0
    t = m.Table.from_columns([_column(m, m.INT32, p, False), _column(m, dt, o, nullable, scale), _column(m, m.INT64, vals["i64"], nullable),
                              _column(m, m.FLOAT64, vals["f64"], nullable), _column(m, m.DECIMAL64, vals["d18"], nullable, 2)])
    srt = m.order_by(t, [(0, 1, 1), (1, asc, nulls_first)])
    return srt, srt.to_pylists()


def _check(m, srt, cols, frames, asc, nulls_first, part_by=(0,), only=None):
    """b2_window over every frame x function (only: the indexes of _funcs to run) against the oracle, frames computed once per
    (lower, upper)"""
    funcs = []
    for fr in frames:
        funcs += [(fr,) + f for j, f in enumerate(_funcs(m, fr, 2)) if only is None or j in only]
    order = [(1, asc, nulls_first)]
    out = m.window(srt, list(part_by), order, [f[1] for f in funcs])
    pk = list(zip(*[cols[c] for c in part_by])) if part_by else [()] * srt.num_rows
    ok = [(x,) for x in cols[1]]
    names = {"i64": 2, "f64": 3, "d18": 4}
    fcache = {}
    for k, (fr, _, kind, col, vt) in enumerate(funcs):
        if fr not in fcache:
            fcache[fr] = R.frames(pk, ok, fr[0], fr[1], bool(asc), bool(nulls_first))
        exp = R.aggregate(fcache[fr], kind, cols[names[col]] if col else None, vt, fr == (None, 0), 28)
        got = out.column(5 + k).to_pylist()
        assert _same(got, exp), (fr, kind, col, [(i, g, e) for i, (g, e) in enumerate(zip(got, exp)) if not _same([g], [e])][:5])
    return out


@pytest.mark.parametrize("asc,nulls_first", [(1, 1), (1, 0), (0, 1), (0, 0)])
@pytest.mark.parametrize("otype", list(ORDER_POOLS))
def test_every_order_type_and_direction_matches_the_oracle(b2, otype, asc, nulls_first):
    m = b2
    pool, ks = ORDER_POOLS[otype]
    nullable = (asc + nulls_first) % 2 == 0
    rng = np.random.default_rng(list(ORDER_POOLS).index(otype) * 4 + asc * 2 + nulls_first)
    srt, cols = _sorted_table(m, rng, 300, 3, otype, pool, asc, nulls_first, nullable)
    _check(m, srt, cols, _frames(ks), asc, nulls_first)


@pytest.mark.parametrize("n,nparts", [(0, 1), (1, 1), (TILE - 1, 2), (TILE, 1), (TILE + 1, 3), (3 * TILE + 3, 3)])
def test_table_sizes_and_partitions_across_tiles(b2, n, nparts):
    """order values of ~4 rows each, so frames of k = 40 span ~160 rows and cross tiles; UNBOUNDED sides span partitions of
    several tiles"""
    m = b2
    rng = np.random.default_rng(n + 7)
    pool = list(range(0, max(n // 4, 1) * 3, 3))
    srt, cols = _sorted_table(m, rng, n, nparts, "INT32", pool, 1, 1, True)
    _check(m, srt, cols, [(-40, 40), (1, 3), (-40, None), (None, 40), (0, 0)], 1, 1, only=(1, 2, 4, 5, 6))


def test_aliases_equal_range_frames_and_launch_no_bounds_kernel(b2):
    m = b2
    rng = np.random.default_rng(3)
    srt, cols = _sorted_table(m, rng, 3 * TILE + 5, 4, "INT64", ORDER_POOLS["INT64"][0], 0, 0, True)
    order = [(1, 0, 0)]
    for lo, up in ((None, 0), (None, None)):
        new = [f for f, _, _, _ in _funcs(m, (lo, up), 2)]
        old = [m.WindowFunc(f.kind, f.column, m.Frame(m.FRAME_RANGE, lo, up), out_dtype=f.out_dtype, out_precision=f.out_precision) for f in new]
        got, names = _kernels(m, lambda: m.window(srt, [0], order, new).to_pylists())
        assert _same_rows(got, m.window(srt, [0], order, old).to_pylists())
        assert "window_range_bounds_kernel" not in names and "window_range_finish_kernel" not in names, names


@pytest.mark.parametrize("case", ["two_columns", "string"])
def test_current_row_bounds_over_any_order_by(b2, case):
    m = b2
    rng = np.random.default_rng(13)
    n = 2 * TILE + 11
    p = [int(x) for x in rng.integers(0, 5, n)]
    a = [None if rng.random() < 0.1 else int(x) for x in rng.integers(0, 4, n)]
    s = [None if rng.random() < 0.1 else "k%d" % int(x) for x in rng.integers(0, 9, n)]
    v = [None if rng.random() < 0.1 else float(x) for x in rng.integers(-50, 50, n)]
    t = m.Table.from_columns([_column(m, m.INT32, p, False), _column(m, m.INT16, a, True), m.Column.from_strings(s), _column(m, m.FLOAT64, v, True)])
    order = [(1, 1, 0), (2, 0, 1)] if case == "two_columns" else [(2, 0, 0)]
    srt = m.order_by(t, [(0, 1, 1)] + order)
    cols = srt.to_pylists()
    pk = [(x,) for x in cols[0]]
    ok = list(zip(*[cols[c] for c, _, _ in order]))
    for lo, up in ((0, 0), (0, None), (None, 0), (None, None)):
        fr = m.range_between(lo, up)
        funcs = [m.win_sum(3, fr), m.win_min(3, fr), m.win_max(1, fr), m.win_count_all(fr)]
        out, names = _kernels(m, lambda: m.window(srt, [0], order, funcs))
        assert ("window_range_bounds_kernel" in names) == (lo == 0), names
        frs = R.frames(pk, ok, lo, up)
        for k, (kind, c, vt) in enumerate(((W.SUM, 3, "float"), (W.MIN, 3, "float"), (W.MAX, 1, "int"), (W.COUNT_ALL, None, "int"))):
            exp = R.aggregate(frs, kind, cols[c] if c is not None else None, vt, lo is None and up == 0)
            assert _same(out.column(4 + k).to_pylist(), exp), (lo, up, kind)


def test_frame_width_does_not_set_the_work_per_row(b2):
    """2^22 rows, one partition, 4 order values of 2^20 rows each: RANGE BETWEEN 1 PRECEDING AND 1 FOLLOWING holds up to 3 * 2^20
    rows, so a loop over each frame would read ~10^13 values.  Checked against numpy closed forms per order value."""
    m = b2
    n, g = 1 << 22, 1 << 20
    o = np.repeat(np.arange(4, dtype=np.int32), g)
    rng = np.random.default_rng(29)
    x = rng.integers(-500, 500, n).astype(np.int64)
    t = m.Table.from_columns([m.Column.from_numpy(o), m.Column.from_numpy(x), m.Column.from_numpy(x.astype(np.float64))])
    fr = m.range_between(-1, 1)
    out, names = _kernels(m, lambda: m.window(t, [], [(0, 1, 1)], [m.win_min(1, fr), m.win_max(1, fr), m.win_sum(2, fr)]))
    assert {"window_range_bounds_kernel", "window_range_tiles_kernel", "window_range_table_kernel", "window_range_finish_kernel"} <= names, names
    groups = x.reshape(4, g)
    for k in range(4):
        sl = groups[max(0, k - 1):k + 2]
        rows = slice(k * g, (k + 1) * g)
        assert np.all(out.column(3).to_numpy()[0][rows] == sl.min())
        assert np.all(out.column(4).to_numpy()[0][rows] == sl.max())
        assert np.all(out.column(5).to_numpy()[0][rows] == float(sl.sum()))


@pytest.mark.parametrize("partitioned", [True, False])
@pytest.mark.parametrize("nbatches", [1, 2, 9, 40])
def test_exec_equals_one_batch(b2, nbatches, partitioned):
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(nbatches * 10 + partitioned)
    n = 3 * TILE + 17
    srt, _ = _sorted_table(m, rng, n, 6 if partitioned else 1, "DATE32", list(range(0, 400, 2)), 0, 1, True)
    parts = [0] if partitioned else []
    order = [(1, 0, 1)]
    funcs = [m.win_sum(2, m.range_between(-7, 0)), m.win_max(3, m.range_between(-7, 7)), m.win_min(3, m.range_between(1, 3)),
             m.win_sum(4, m.range_between(-20, None), m.DECIMAL128, 28), m.win_count_all(m.range_between(0, 0)), m.win_sum(3, m.range_between(None, 0)),
             m.rank(), m.lag(2, 2)]
    exp = m.window(srt, parts, order, funcs).to_pylists()
    cuts = sorted(set(int(x) for x in rng.integers(0, n, nbatches - 1)))   # inside partitions and peer groups
    cuts = sorted(cuts + cuts[:2])                                          # repeated cuts: empty batches
    ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, srt, cuts)), parts, order, funcs)
    got = [[] for _ in exp]
    for b in ex:
        for c, vals in enumerate(b.to_pylists()):
            got[c] += vals
    assert _same_rows(got, exp)
    assert ex.metrics["numOutputRows"] == n


def test_argument_errors(b2):
    m = b2
    t = m.Table.from_columns([_column(m, m.INT32, [1, 1], False), _column(m, m.INT64, [1, 2], False), m.Column.from_strings(["a", "b"]),
                              _column(m, m.FLOAT64, [1.0, 2.0], False), m.Column.from_numpy(np.array([0, 1], dtype=np.int8), m.BOOL8),
                              _column(m, m.DECIMAL128, [1, 2], False, 2), _column(m, m.FLOAT32, [1.0, 2.0], False)])
    rv = m.range_between
    cases = [
        ([], m.win_sum(1, rv(-1, 0)), INVALID),                      # no ORDER BY, a bound other than UNBOUNDED
        ([], m.win_sum(1, rv(None, 0)), INVALID),
        ([(1, 1, 1)], m.win_sum(1, rv(2, 1)), INVALID),             # lower > upper
        ([(1, 1, 1)], m.win_sum(1, m.Frame(m.FRAME_RANGE_VALUE, m.UNBOUNDED_FOLLOWING, None)), INVALID),   # wrong direction
        ([(1, 1, 1), (0, 1, 1)], m.win_sum(1, rv(-1, 0)), INVALID),  # offsets need one ORDER BY column
        ([(2, 1, 1)], m.win_count_all(rv(-1, 1)), INVALID),         # STRING
        ([(4, 1, 1)], m.win_count_all(rv(0, 1)), INVALID),          # BOOL8
        ([(3, 1, 1)], m.win_count_all(rv(-1, 0)), UNSUPPORTED),     # FLOAT64
        ([(6, 1, 1)], m.win_count_all(rv(-1, 0)), UNSUPPORTED),     # FLOAT32
        ([(1, 1, 1)], m.win_min(2, rv(-1, 1)), UNSUPPORTED),        # MIN over STRING
        ([(1, 1, 1)], m.win_max(5, rv(-1, 1)), UNSUPPORTED),        # MAX over DECIMAL128
    ]
    for order, f, code in cases:
        with pytest.raises(m.B2Error) as ei:
            m.window(t, [0], order, [f])
        assert ei.value.code == code, (order, f.frame.lower, f.frame.upper, ei.value)
    # without ORDER BY the whole partition is fine, and CURRENT ROW bounds need no value type
    assert m.window(t, [0], [], [m.win_count_all(rv(None, None))]).column(7).to_pylist() == [2, 2]
    assert m.window(t, [0], [(2, 1, 1), (3, 0, 1)], [m.win_count_all(rv(0, None))]).column(7).to_pylist() == [2, 1]
