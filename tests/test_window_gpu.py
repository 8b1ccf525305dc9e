"""Window functions on the GPU (b2_window, GpuWindowExec) against the row-at-a-time oracle (oracle/spark_window.py): exact for
every function except float SUM, which is a parallel scan: bit for bit where every partial sum is exact in double (NaN and
+-inf included), within a relative bound on random doubles."""
import gc
import math
import struct

import numpy as np
import pytest

from oracle import spark_window as W

pytestmark = pytest.mark.gpu

TILE = 1024   # rows per scan tile (window.cu WIN_TILE)


def _col(m, dtype, vals, scale=0):
    valid = np.array([v is not None for v in vals], dtype=bool)
    if dtype == m.STRING:
        return m.Column.from_strings(vals)
    if dtype == m.DECIMAL128:
        return m.Column.from_numpy(np.array([v if v is not None else 0 for v in vals], dtype=object), dtype, valid, scale)
    fill = 0.0 if dtype in (m.FLOAT32, m.FLOAT64) else 0
    return m.Column.from_numpy(np.array([v if v is not None else fill for v in vals]), dtype, valid, scale)


def _sorted_input(rng, n, nparts, dtype_vals=None):
    """n rows sorted by (p, o): p in [0, nparts), o in [0, 6) (ties), plus value columns of each kind"""
    p = np.sort(rng.integers(0, max(nparts, 1), n))
    o = np.zeros(n, dtype=np.int64)
    for g in np.unique(p):
        idx = np.nonzero(p == g)[0]
        o[idx] = np.sort(rng.integers(0, 6, len(idx)))
    ints = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-2**62, 2**62, n)]
    flts = [None if rng.random() < 0.1 else float(x) for x in rng.integers(-1000, 1000, n)]   # sums exact in double
    big = 10 ** 38 - 1
    d38 = [None if rng.random() < 0.1 else int(rng.choice([big, -big, 1, -1, 12345])) for _ in range(n)]
    d18 = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-10**17, 10**17, n)]
    strs = [None if rng.random() < 0.1 else "s%d" % int(x) for x in rng.integers(0, 50, n)]
    return [int(x) for x in p], [int(x) for x in o], {"i64": ints, "f64": flts, "d38": d38, "d18": d18, "str": strs}


def _table(m, p, o, vals):
    return m.Table.from_columns([_col(m, m.INT32, p), _col(m, m.INT64, o), _col(m, m.INT64, vals["i64"]), _col(m, m.FLOAT64, vals["f64"]),
                                 _col(m, m.DECIMAL128, vals["d38"], 2), _col(m, m.DECIMAL64, vals["d18"], 2), _col(m, m.STRING, vals["str"])])


COLS = {"i64": (2, "int"), "f64": (3, "float"), "d38": (4, "decimal"), "d18": (5, "decimal")}
FRAMES = [(W.ROWS, None, 0), (W.RANGE, None, 0), (W.ROWS, None, None), (W.ROWS, -3, 2), (W.ROWS, -5, -1), (W.ROWS, 1, 4), (W.ROWS, 0, 0),
          (W.ROWS, -700, 700), (W.ROWS, None, 2), (W.ROWS, -2, None)]


def _funcs(m):
    """(WindowFunc, oracle kwargs) for every function x frame over every value column"""
    out = [(m.row_number(), dict(kind=W.ROW_NUMBER)), (m.rank(), dict(kind=W.RANK)), (m.dense_rank(), dict(kind=W.DENSE_RANK))]
    for off in (0, 1, 5, 3000):
        out.append((m.lead(6, off), dict(kind=W.LEAD, col="str", offset=off)))
        out.append((m.lag(2, off, default=-7), dict(kind=W.LAG, col="i64", offset=off, default=-7)))
        out.append((m.lag(3, off, default=2.5, dtype=m.FLOAT64), dict(kind=W.LAG, col="f64", offset=off, default=2.5)))
    for ft, lo, up in FRAMES:
        fr = m.Frame(ft, lo, up)
        kw = dict(frame=ft, lower=lo, upper=up)
        for name, (c, vt) in COLS.items():
            if vt == "decimal":
                prec = 38 if name == "d38" else 28
                out.append((m.win_sum(c, fr, m.DECIMAL128, prec), dict(kind=W.SUM, col=name, vtype=vt, precision=prec, **kw)))
            else:
                out.append((m.win_sum(c, fr), dict(kind=W.SUM, col=name, vtype=vt, **kw)))
            out.append((m.win_count(c, fr), dict(kind=W.COUNT, col=name, **kw)))
            if name != "d38":
                out.append((m.win_min(c, fr), dict(kind=W.MIN, col=name, vtype=vt, **kw)))
                out.append((m.win_max(c, fr), dict(kind=W.MAX, col=name, vtype=vt, **kw)))
        out.append((m.win_count_all(fr), dict(kind=W.COUNT_ALL, **kw)))
    return out


def _expected(p, o, vals, kw):
    kw = dict(kw)
    col = kw.pop("col", None)
    return W.evaluate([(x,) for x in p], [(x,) for x in o], values=vals[col] if col else None, **kw)


def _same(got, exp, rel=None):
    """exact: every float bit for bit (any NaN matches any NaN); rel: finite floats within that relative bound, +-inf equal"""
    if len(got) != len(exp):
        return False
    for g, e in zip(got, exp):
        if isinstance(e, float) and isinstance(g, float):
            if math.isnan(e) or math.isnan(g):
                if not (math.isnan(e) and math.isnan(g)):
                    return False
            elif rel is None or math.isinf(e) or math.isinf(g):
                if struct.pack("<d", g) != struct.pack("<d", e):
                    return False
            elif abs(g - e) > rel * max(1.0, abs(e)):
                return False
        elif type(g) is not type(e) or g != e:
            return False
    return True


def _check_all(m, p, o, vals, funcs=None):
    funcs = funcs or _funcs(m)
    t = _table(m, p, o, vals)
    out = m.window(t, [0], [(1, 1, 1)], [f for f, _ in funcs])
    assert out.num_columns == 7 + len(funcs)
    for k, (f, kw) in enumerate(funcs):
        got = out.column(7 + k).to_pylist()
        exp = _expected(p, o, vals, kw)
        assert _same(got, exp), (kw, [(i, g, e) for i, (g, e) in enumerate(zip(got, exp)) if not _same([g], [e])][:5])
    return out


@pytest.mark.parametrize("n,nparts", [(0, 1), (1, 1), (TILE - 1, 7), (TILE, 1), (TILE + 1, 3), (3 * TILE + 5, 40), (4 * TILE, 3)])
def test_every_function_and_frame_matches_the_oracle(b2, n, nparts):
    rng = np.random.default_rng(n + nparts)
    p, o, vals = _sorted_input(rng, n, nparts)
    _check_all(b2, p, o, vals)


def test_partition_start_on_a_tile_boundary_and_one_row_partitions(b2):
    m = b2
    n = 3 * TILE
    p = [0] * TILE + list(range(1, TILE + 1)) + [TILE + 1] * TILE
    o = [i % 4 for i in range(n)]
    o = [x for _, x in sorted(zip(p, o))]
    rng = np.random.default_rng(5)
    _, _, vals = _sorted_input(rng, n, 1)
    _check_all(m, p, o, vals)


def test_float_sum_nan_inf_and_signed_zero(b2):
    m = b2
    p = [0] * 6 + [1] * 4
    o = list(range(10))
    f = [1.0, math.inf, 2.0, -math.inf, 3.0, None, -0.0, 0.0, math.nan, 1.0]
    vals = {"i64": [0] * 10, "f64": f, "d38": [0] * 10, "d18": [0] * 10, "str": ["a"] * 10}
    funcs = [(m.win_sum(3, m.rows(None, 0)), dict(kind=W.SUM, col="f64", vtype="float", lower=None, upper=0)),
             (m.win_sum(3, m.unbounded()), dict(kind=W.SUM, col="f64", vtype="float", lower=None, upper=None)),
             (m.win_sum(3, m.rows(-1, 1)), dict(kind=W.SUM, col="f64", vtype="float", lower=-1, upper=1)),
             (m.win_min(3, m.unbounded()), dict(kind=W.MIN, col="f64", vtype="float", lower=None, upper=None)),
             (m.win_max(3, m.rows(-1, 0)), dict(kind=W.MAX, col="f64", vtype="float", lower=-1, upper=0))]
    _check_all(m, p, o, vals, funcs)


def test_decimal_running_sum_goes_null_and_stays_null(b2):
    m = b2
    big = 10 ** 38 - 1
    n = 2 * TILE + 10
    p = [0] * n
    o = list(range(n))
    d38 = [1] * n
    d38[0], d38[TILE + 3] = big - 5, -(n + 10)   # overflows at row 6 and comes back in range: running stays NULL, the total fits
    vals = {"i64": [0] * n, "f64": [0.0] * n, "d38": d38, "d18": [0] * n, "str": ["a"] * n}
    funcs = [(m.win_sum(4, m.rows(None, 0), m.DECIMAL128, 38), dict(kind=W.SUM, col="d38", vtype="decimal", lower=None, upper=0)),
             (m.win_sum(4, m.unbounded(), m.DECIMAL128, 38), dict(kind=W.SUM, col="d38", vtype="decimal", lower=None, upper=None))]
    out = _check_all(m, p, o, vals, funcs)
    run = out.column(7).to_pylist()
    assert run[5] == big and all(v is None for v in run[6:])
    assert out.column(8).to_pylist() == [big - 17] * n


def test_keys_of_every_kind_nan_zero_null_form_one_group(b2):
    m = b2
    # float partition key: NULL, NaN (two payloads), -0.0 / 0.0; string order key DESC nulls last
    pk = [None, None, math.nan, -math.nan, -0.0, 0.0, 1.5]
    ok = ["b", "a", "b", "b", "c", None, "x"]
    t = m.Table.from_columns([_col(m, m.FLOAT64, pk), _col(m, m.STRING, ok)])
    out = m.window(t, [0], [(1, 0, 0)], [m.row_number(), m.rank(), m.dense_rank()])
    assert out.column(2).to_pylist() == [1, 2, 1, 2, 1, 2, 1]
    assert out.column(3).to_pylist() == [1, 2, 1, 1, 1, 2, 1]
    assert out.column(4).to_pylist() == [1, 2, 1, 1, 1, 2, 1]


def test_whole_partition_aggregates_equal_groupby(b2):
    m = b2
    rng = np.random.default_rng(11)
    p, o, vals = _sorted_input(rng, 4 * TILE, 30)
    t = _table(m, p, o, vals)
    fr = m.unbounded()
    out = m.window(t, [0], [(1, 1, 1)], [m.win_sum(2, fr), m.win_count(2, fr), m.win_min(2, fr), m.win_max(2, fr), m.win_sum(5, fr, m.DECIMAL128, 28)])
    g = m.groupby(t, [0], [(m.AGG_SUM, 2, m.INT64), (m.AGG_COUNT, 2, m.INT64), (m.AGG_MIN, 2, m.INT64), (m.AGG_MAX, 2, m.INT64),
                           (m.AGG_SUM, 5, m.DECIMAL128, 2, 28)])
    by_key = {r[0]: r[1:] for r in g.to_rows()}
    for r in out.to_rows():
        assert tuple(r[7:]) == tuple(by_key[r[0]])


def test_argument_errors(b2):
    m = b2
    t = m.Table.from_columns([_col(m, m.INT32, [1, 1]), _col(m, m.INT64, [1, 2]), _col(m, m.STRING, ["a", "b"])])
    cases = [([], m.rank(), 1), ([(1, 1, 1)], m.WindowFunc(m.WIN_SUM, 1, m.Frame(m.FRAME_RANGE, -1, 0)), 5),
             ([(1, 1, 1)], m.win_min(2, m.unbounded()), 5), ([(1, 1, 1)], m.lag(2, 1, default=3), 5),
             ([(1, 1, 1)], m.win_sum(1, m.rows(2, 1)), 1), ([(1, 1, 1)], m.win_sum(9, m.unbounded()), 1),
             ([], m.lead(1, 1), 1)]
    for order, f, code in cases:
        with pytest.raises(m.B2Error) as ei:
            m.window(t, [0], order, [f])
        assert ei.value.code == code, (f.kind, ei.value)


def _kernels(m, fn):
    m.profile_enable(True)
    try:
        r = fn()
        names = {k["name"] for k in m.profile_report()}
    finally:
        m.profile_enable(False)
    return r, names


def _batches(m, t, cuts):
    out = []
    prev = 0
    for c in list(cuts) + [t.num_rows]:
        out.append(m.slice_table(t, prev, c))
        prev = c
    return out


MODE_FUNCS = {
    1: lambda m: [m.row_number(), m.rank(), m.dense_rank(), m.win_sum(2, m.rows(None, 0)), m.win_sum(4, m.rows(None, 0), m.DECIMAL128, 38),
                  m.win_count(3, m.rows(None, 0)), m.win_min(2, m.rows(None, 0)), m.win_max(3, m.rows(None, 0))],
    2: lambda m: [m.rank(), m.win_sum(2, m.range_running()), m.win_sum(5, m.range_running(), m.DECIMAL128, 28), m.win_count_all(m.range_running())],
    3: lambda m: [m.win_sum(2, m.unbounded()), m.win_sum(2, m.rows(-6, 0)), m.lag(2, 1), m.lead(6, 2), m.win_min(3, m.rows(-2, 2)), m.row_number()],
}


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("nbatches", [1, 2, 7, 40])
def test_exec_equals_one_batch(b2, mode, nbatches):
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(mode * 100 + nbatches)
    n = 3 * TILE + 17
    p, o, vals = _sorted_input(rng, n, 5 if mode != 1 else 60)
    t = _table(m, p, o, vals)
    funcs = MODE_FUNCS[mode](m)
    exp = m.window(t, [0], [(1, 1, 1)], funcs).to_rows()
    cuts = sorted(set(int(x) for x in rng.integers(0, n, nbatches - 1)))   # repeated cuts give empty batches
    cuts = sorted(cuts + cuts[:2])
    ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, t, cuts)), [0], [(1, 1, 1)], funcs)
    got, names = _kernels(m, lambda: [b.to_rows() for b in ex])
    assert [r for b in got for r in b] == exp
    assert "window_scan_kernel" in names and "window_bounds_kernel" in names
    assert ("window_group_ends_kernel" in names) == (mode != 1)
    assert ("window_last_start_kernel" in names) == (mode != 1)
    mt = ex.metrics
    assert mt["numOutputRows"] == n
    if mode == 1:
        assert mt["numOutputBatches"] == len([1 for a, b in zip([0] + cuts, cuts + [n]) if b > a])


def test_exec_over_unsorted_input_through_sort(b2):
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(9)
    n = 2 * TILE + 3
    p, o, vals = _sorted_input(rng, n, 20)
    perm = rng.permutation(n)
    t = _table(m, p, o, vals)
    shuffled = m.gather(t, m.Column.from_numpy(perm.astype(np.int32)))
    funcs = [m.rank(), m.win_sum(2, m.range_running()), m.win_count(2, m.unbounded())]
    srt = E.GpuSortExec([(0, 1, 1), (1, 1, 1)], E.GpuBatchSource(_batches(m, shuffled, [100, 900, 1500])))
    out = E.GpuWindowExec(srt, [0], [(1, 1, 1)], funcs).collect()
    got = out.to_rows()
    exp_rank = _expected(p, o, vals, dict(kind=W.RANK))
    exp_sum = _expected(p, o, vals, dict(kind=W.SUM, col="i64", frame=W.RANGE, lower=None, upper=0))
    assert [r[7] for r in got] == exp_rank
    assert [r[8] for r in got] == exp_sum
    assert [(r[0], r[1]) for r in got] == list(zip(p, o))


# ---- every key and value type ---------------------------------------------------------------------------------------------------
BIG = {9: 10 ** 9 - 1, 18: 10 ** 18 - 1, 38: 10 ** 38 - 1}


def _f32_nan(payload):
    return float(np.array([0x7FC00000 | payload], dtype=np.uint32).view(np.float32)[0])


def _f64_nan(payload):
    return float(np.array([0x7FF8000000000000 | payload], dtype=np.uint64).view(np.float64)[0])


def _values(m, rng, dtype, n, nullable, keys=False):
    """random values of one type: few distinct ones for keys (so groups form), edge values for value columns"""
    if dtype == m.STRING:
        pool = ["", "a", "ab", "b", "été"] if keys else ["s%d" % i for i in range(40)]
    elif dtype in (m.FLOAT32, m.FLOAT64):
        nan = _f32_nan if dtype == m.FLOAT32 else _f64_nan
        pool = [nan(0), nan(5), -0.0, 0.0, 1.5, -math.inf] if keys else [nan(0), nan(7), math.inf, -math.inf, -0.0, 0.0] + [float(x) for x in range(-60, 60)]
    elif dtype in (m.DECIMAL32, m.DECIMAL64, m.DECIMAL128):
        big = BIG[{m.DECIMAL32: 9, m.DECIMAL64: 18, m.DECIMAL128: 38}[dtype]]
        pool = [big, -big, 0, 1, -7] if keys else [big, -big, 1, -1, 12345, -99999]
    else:
        bits = {m.INT8: 8, m.INT16: 16, m.INT32: 32, m.INT64: 64, m.DATE32: 20, m.TIMESTAMP_US: 50}[dtype]
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        pool = [lo, hi, 0, 3, -3] if keys else [lo, hi, 0] + [int(x) for x in rng.integers(lo // 2, hi // 2, 40)]
    vals = [pool[int(i)] for i in rng.integers(0, len(pool), n)]
    if nullable:
        vals = [None if rng.random() < 0.15 else v for v in vals]
    return vals


def _column(m, dtype, vals, nullable, scale=0):
    if dtype == m.STRING:
        return m.Column.from_strings(vals)
    valid = np.array([v is not None for v in vals], dtype=bool) if nullable else None
    if dtype == m.DECIMAL128:
        return m.Column.from_numpy(np.array([v if v is not None else 0 for v in vals], dtype=object), dtype, valid, scale)
    np_t = {m.FLOAT32: np.float32, m.FLOAT64: np.float64}.get(dtype, np.int64)
    return m.Column.from_numpy(np.array([v if v is not None else 0 for v in vals], dtype=np_t), dtype, valid, scale)


VALUE_TYPES = ["INT8", "INT16", "INT32", "INT64", "DATE32", "FLOAT32", "FLOAT64", "DECIMAL32", "DECIMAL64", "DECIMAL128", "STRING"]
PREC = {"DECIMAL32": 9, "DECIMAL64": 18, "DECIMAL128": 38}


def _value_funcs(m, name, c):
    """(WindowFunc, oracle kwargs, runs in mode 1) for a value column of type `name` at index c"""
    dt = getattr(m, name)
    vt = "float" if name.startswith("FLOAT") else "decimal" if name.startswith("DECIMAL") else "int" if name.startswith("INT") else "other"
    default = None if name == "STRING" else 1.5 if vt == "float" else 2
    out = [(m.lag(c, 1, default=default, dtype=dt if vt == "float" else None), dict(kind=W.LAG, offset=1, default=default), False),
           (m.lead(c, 3), dict(kind=W.LEAD, offset=3), False)]
    for fr, run in ((m.rows(None, 0), True), (m.range_running(), False), (m.unbounded(), False), (m.rows(-3, 2), False), (m.rows(1, 4), False)):
        kw = dict(frame=fr.type, lower=fr.lower, upper=fr.upper)
        out.append((m.win_count(c, fr), dict(kind=W.COUNT, **kw), run))
        if vt in ("int", "float"):
            out.append((m.win_sum(c, fr), dict(kind=W.SUM, vtype=vt, **kw), run))
        if vt == "decimal":
            p = min(38, PREC[name] + 10)
            out.append((m.win_sum(c, fr, m.DECIMAL128, p), dict(kind=W.SUM, vtype=vt, precision=p, **kw), run))
        if name not in ("STRING", "DECIMAL128"):
            out.append((m.win_min(c, fr), dict(kind=W.MIN, vtype=vt, **kw), run))
            out.append((m.win_max(c, fr), dict(kind=W.MAX, vtype=vt, **kw), run))
    return out


KEY_CASES = [   # (partition key types, order keys as (type, ascending, nulls_first))
    (["INT32"], [("INT64", 1, 1)]),
    (["INT8", "STRING"], [("FLOAT64", 0, 0), ("INT16", 1, 0)]),
    (["FLOAT32"], [("DECIMAL128", 0, 1)]),
    (["DATE32", "DECIMAL32"], [("STRING", 1, 1), ("TIMESTAMP_US", 0, 0)]),
    (["DECIMAL64"], [("FLOAT32", 1, 0)]),
    ([], [("INT32", 0, 1), ("STRING", 0, 0)]),
]


def _matrix_case(m, seed, parts, orders, nullable, n):
    """an unsorted random table (keys, then one column per value type), sorted on the GPU by (partition, order)"""
    rng = np.random.default_rng(seed)
    key_types = parts + [t for t, _, _ in orders]
    cols, data = [], []
    for i, name in enumerate(key_types):
        v = _values(m, rng, getattr(m, name), n, nullable and i % 2 == 0, keys=True)
        cols.append(_column(m, getattr(m, name), v, nullable and i % 2 == 0, 2 if name.startswith("DECIMAL") else 0))
    for name in VALUE_TYPES:
        v = _values(m, rng, getattr(m, name), n, nullable)
        cols.append(_column(m, getattr(m, name), v, nullable, 2 if name.startswith("DECIMAL") else 0))
    t = m.Table.from_columns(cols)
    np_ = len(parts)
    part_cols = list(range(np_))
    order = [(np_ + i, a, nf) for i, (_, a, nf) in enumerate(orders)]
    srt = m.order_by(t, [(c, 1, 1) for c in part_cols] + order)
    return srt, part_cols, order, len(key_types)


def _oracle_inputs(srt, part_cols, order):
    cols = srt.to_pylists()
    pk = list(zip(*[cols[c] for c in part_cols])) if part_cols else [()] * srt.num_rows
    ok = list(zip(*[cols[c] for c, _, _ in order]))
    return cols, pk, ok


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("case", range(len(KEY_CASES)))
def test_every_key_and_value_type(b2, case, nullable):
    """b2_window, and GpuWindowExec over 9 batches (mode 1: the running functions, carried across batches; mode 3: all of
    them), against the oracle over the GPU-sorted rows"""
    m = b2
    from spark_rapids_b200 import execs as E
    parts, orders = KEY_CASES[case]
    n = 2 * TILE + 37
    srt, part_cols, order, nkeys = _matrix_case(m, 40 + case, parts, orders, nullable, n)
    cols, pk, ok = _oracle_inputs(srt, part_cols, order)
    funcs = []
    for j, name in enumerate(VALUE_TYPES):
        for f, kw, run in _value_funcs(m, name, nkeys + j):
            funcs.append((f, kw, run, nkeys + j))
    funcs += [(m.row_number(), dict(kind=W.ROW_NUMBER), True, None), (m.rank(), dict(kind=W.RANK), True, None),
              (m.dense_rank(), dict(kind=W.DENSE_RANK), True, None)]
    out = m.window(srt, part_cols, order, [f for f, _, _, _ in funcs])
    base = srt.num_columns
    expected = []
    for k, (f, kw, _, c) in enumerate(funcs):
        exp = W.evaluate(pk, ok, values=cols[c] if c is not None else None, **kw)
        expected.append(exp)
        got = out.column(base + k).to_pylist()
        assert _same(got, exp), (k, kw, [(i, g, e) for i, (g, e) in enumerate(zip(got, exp)) if not _same([g], [e])][:5])
    cuts = sorted(int(x) for x in np.random.default_rng(case).integers(0, n, 8))
    for mode1 in (True, False):
        sel = [k for k, (_, _, run, _) in enumerate(funcs) if run or not mode1]
        ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, srt, cuts)), part_cols, order, [funcs[k][0] for k in sel])
        batches = list(ex)
        got_cols = [[] for _ in sel]
        for b in batches:
            for i in range(len(sel)):
                got_cols[i] += b.column(base + i).to_pylist()
        for i, k in enumerate(sel):
            assert _same(got_cols[i], expected[k]), (mode1, funcs[k][1])


def test_float_sum_of_random_doubles_within_a_relative_bound(b2):
    m = b2
    rng = np.random.default_rng(17)
    n = 3 * TILE + 9
    p = sorted(int(x) for x in rng.integers(0, 4, n))
    f = [float(x) for x in rng.normal(0, 1e6, n)]
    f[5], f[2000] = math.inf, -math.inf   # partition 0 (or 1) gets +inf, a later one -inf: inf - inf = NaN only where both meet
    t = m.Table.from_columns([_col(m, m.INT32, p), _col(m, m.INT64, list(range(n))), _col(m, m.FLOAT64, f)])
    frames = [m.rows(None, 0), m.range_running(), m.unbounded(), m.rows(-5, 5)]
    out = m.window(t, [0], [(1, 1, 1)], [m.win_sum(2, fr) for fr in frames])
    for k, fr in enumerate(frames):
        exp = W.evaluate([(x,) for x in p], [(i,) for i in range(n)], W.SUM, f, vtype="float", frame=fr.type, lower=fr.lower, upper=fr.upper)
        assert _same(out.column(3 + k).to_pylist(), exp, rel=1e-9), k


@pytest.mark.parametrize("name", [t for t in VALUE_TYPES if t != "STRING"])
def test_whole_partition_aggregates_equal_groupby_for_every_type(b2, name):
    m = b2
    n = 3 * TILE
    srt, part_cols, order, nkeys = _matrix_case(m, 77, ["INT32"], [("INT64", 1, 1)], True, n)
    fr = m.unbounded()
    c, dt = nkeys + VALUE_TYPES.index(name), getattr(m, name)
    funcs, aggs = [m.win_count(c, fr)], [(m.AGG_COUNT, c, m.INT64)]
    if name.startswith("INT") or name.startswith("FLOAT"):
        funcs.append(m.win_sum(c, fr)); aggs.append((m.AGG_SUM, c, m.FLOAT64 if name.startswith("FLOAT") else m.INT64))
    if name.startswith("DECIMAL"):
        p = min(38, PREC[name] + 10)
        funcs.append(m.win_sum(c, fr, m.DECIMAL128, p)); aggs.append((m.AGG_SUM, c, m.DECIMAL128, 2, p))
    if name != "DECIMAL128":
        funcs.append(m.win_min(c, fr)); aggs.append((m.AGG_MIN, c, dt))
        funcs.append(m.win_max(c, fr)); aggs.append((m.AGG_MAX, c, dt))
    out = m.window(srt, part_cols, order, funcs)
    g = m.groupby(srt, part_cols, aggs)
    gcols = g.to_pylists()
    by_key = {gcols[0][r]: [gcols[1 + k][r] for k in range(len(aggs))] for r in range(g.num_rows)}
    ocols = out.to_pylists()
    base = srt.num_columns
    for r in range(out.num_rows):
        got = [ocols[base + k][r] for k in range(len(funcs))]
        assert _same(got, by_key[ocols[0][r]]), (r, got, by_key[ocols[0][r]])


# ---- AVG, split-and-retry, spill ------------------------------------------------------------------------------------------------
def test_avg_is_sum_over_count_through_a_projection(b2):
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(23)
    n = 2 * TILE + 5
    p = sorted(int(x) for x in rng.integers(0, 9, n))
    v = [None if rng.random() < 0.3 else int(x) for x in rng.integers(-1000, 1000, n)]
    t = m.Table.from_columns([_col(m, m.INT32, p), _col(m, m.INT64, list(range(n))), _col(m, m.INT64, v)])
    frames = [m.rows(-6, 0), m.unbounded(), m.range_running()]
    funcs = []
    for fr in frames:
        funcs += [m.win_sum(2, fr), m.win_count(2, fr)]
    win = E.GpuWindowExec(E.GpuBatchSource(_batches(m, t, [300, 1200])), [0], [(1, 1, 1)], funcs)
    avg = [m.col(3 + 2 * k, m.INT64).cast(m.FLOAT64) / m.col(4 + 2 * k, m.INT64).cast(m.FLOAT64) for k in range(len(frames))]
    out = E.GpuProjectExec(avg, win).collect()
    for k, fr in enumerate(frames):
        kw = dict(frame=fr.type, lower=fr.lower, upper=fr.upper)
        s = W.evaluate([(x,) for x in p], [(i,) for i in range(n)], W.SUM, v, **kw)
        c = W.evaluate([(x,) for x in p], [(i,) for i in range(n)], W.COUNT, v, **kw)
        exp = [None if cc == 0 else float(ss) / float(cc) for ss, cc in zip(s, c)]
        assert _same(out.column(k).to_pylist(), exp), k


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


def test_running_exec_splits_a_batch_under_an_allocation_limit(b2, limits):
    """mode 1 over one batch of 2^21 rows needs ~61 B per row at its peak; a half, with both halves' copies, ~47 B per row.
    Under a limit of 54 B per row the batch is split, and the halves, continued through the carry, equal the whole"""
    m = b2
    from spark_rapids_b200 import execs as E
    n = 1 << 21
    rng = np.random.default_rng(31)
    key = np.sort(rng.integers(0, 5000, n)).astype(np.int64)
    val = rng.integers(-10**6, 10**6, n).astype(np.int64)
    funcs = [m.row_number(), m.win_sum(1, m.rows(None, 0))]
    t = m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(val)])
    ref = m.window(t, [0], [], funcs[1:])
    exp_sum = ref.column(2).to_numpy()[0]
    del ref
    rn_exp = np.arange(n) - np.searchsorted(key, key, side="left") + 1
    src = E.GpuBatchSource([t])
    del t
    gc.collect()
    m.sync()
    s0 = m.memory_stats()
    m.set_alloc_limit(m.device_bytes_in_use() + 54 * n)
    ex = E.GpuWindowExec(src, [0], [(0, 1, 1)], funcs)
    del src
    rn, sm, nout = [], [], 0
    while True:
        b = ex.next()
        if b is None:
            break
        rn.append(b.column(2).to_numpy()[0]); sm.append(b.column(3).to_numpy()[0]); nout += 1
        del b
    m.set_alloc_limit(0)
    s1 = m.memory_stats()
    assert s1["splits"] > s0["splits"] and nout >= 2, (s0, s1, nout)
    assert np.array_equal(np.concatenate(rn), rn_exp)
    assert np.array_equal(np.concatenate(sm), exp_sum)
    assert ex.metrics["numOutputRows"] == n and ex.metrics["numOutputBatches"] == nout


def test_held_partition_spills_under_an_allocation_limit(b2, limits):
    """mode 3: partition A arrives over 16 batches of 4096 rows; the batch that ends it carries 16 of its rows and the first
    60000 of partition B.  B's rows wait in the spill store while A's pieces are concatenated (+16.8 MB); with B's piece (+15.4 MB)
    that passes the limit of 24 MB over the input, so B's piece leaves the device, and it comes back when B runs.  Rows are 256
    bytes (2 keys + 30 payload columns)"""
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(37)
    sizes = [4096] * 16 + [16 + 60000] + [4096] * 3
    n = sum(sizes)
    part = np.where(np.arange(n) < 16 * 4096 + 16, 0, 1).astype(np.int64)
    cols = [part, np.arange(n, dtype=np.int64)] + [rng.integers(-1000, 1000, n).astype(np.int64) for _ in range(30)]
    funcs = [m.win_sum(2, m.unbounded()), m.row_number(), m.lag(3, 1), m.lead(4, 2), m.win_sum(5, m.rows(-3, 3))]
    whole = m.Table.from_columns([m.Column.from_numpy(c) for c in cols])
    ref = m.window(whole, [0], [(1, 1, 1)], funcs)
    exp = [ref.column(32 + k).to_pylist() for k in range(len(funcs))]
    del ref
    batches, s = [], 0
    for z in sizes:
        batches.append(m.slice_table(whole, s, s + z))
        s += z
    del whole
    src = E.GpuBatchSource(batches)
    del batches
    gc.collect()
    m.sync()
    base = m.device_bytes_in_use()
    s0 = m.memory_stats()
    m.set_alloc_limit(base + (24 << 20))
    ex = E.GpuWindowExec(src, [0], [(1, 1, 1)], funcs)
    del src
    got = [[] for _ in funcs]
    nout = 0
    while True:
        b = ex.next()
        if b is None:
            break
        for k in range(len(funcs)):
            got[k] += b.column(32 + k).to_pylist()
        nout += 1
        del b
    m.set_alloc_limit(0)
    s1 = m.memory_stats()
    assert s1["limit"] == 0
    assert s1["spilled_bytes"] > s0["spilled_bytes"] and s1["unspilled_bytes"] > s0["unspilled_bytes"], (s0, s1)
    assert nout == 2
    for k in range(len(funcs)):
        assert got[k] == exp[k], k
    del ex
    gc.collect()
    m.sync()
    assert m.device_bytes_in_use() <= base
