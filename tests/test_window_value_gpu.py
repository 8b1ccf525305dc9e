"""FIRST / LAST / NTH_VALUE with and without IGNORE NULLS on the GPU (b2_window and GpuWindowExec) against the row-at-a-time
restatement (tests/window_value_oracle.py).  The restatement names the row each result is copied from, and the result is compared
with that row's bytes: floats bit for bit (NaN payloads, -0.0), strings byte for byte, "" apart from NULL."""
import gc

import numpy as np
import pytest

from oracle import spark_window as W
from tests import window_range_oracle as R
from tests import window_value_oracle as V
from tests.test_window_gpu import FRAMES, TILE, _batches, _column, _f32_nan, _f64_nan, _kernels

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = 1, 5
KINDS = [(V.FIRST, 1), (V.LAST, 1), (V.NTH_VALUE, 1), (V.NTH_VALUE, 2), (V.NTH_VALUE, 3), (V.NTH_VALUE, 700)]


def _fn(m, kind, n, c, frame, ign):
    if kind == V.FIRST:
        return m.first_value(c, frame, ign)
    if kind == V.LAST:
        return m.last_value(c, frame, ign)
    return m.nth_value(c, n, frame, ign)


def _raw(a):
    a = np.asarray(a)
    if a.dtype.kind == "f":
        return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)
    return a


def _assert_copied(got, src_col, src_rows, what):
    """got: the result column; src_col: the value column; src_rows: the oracle's source row of each result (None: NULL)"""
    gv, gok = got.to_numpy()
    sv, sok = src_col.to_numpy()
    idx = np.array([-1 if j is None else j for j in src_rows], dtype=np.int64)
    exp_ok = (idx >= 0) & np.asarray(sok, dtype=bool)[np.maximum(idx, 0)] if len(idx) else np.zeros(0, bool)
    bad = np.nonzero(np.asarray(gok, dtype=bool) != exp_ok)[0]
    assert len(bad) == 0, (what, "validity", [(int(i), int(idx[i])) for i in bad[:5]])
    gr, sr = _raw(gv), _raw(sv)
    sel = np.nonzero(exp_ok)[0]
    if len(sel):
        a, b = gr[sel], sr[idx[sel]]
        same = np.all(a == b, axis=tuple(range(1, a.ndim))) if a.ndim > 1 else (a == b)
        bad = sel[~np.asarray(same, dtype=bool)]
        assert len(bad) == 0, (what, "value", [(int(i), int(idx[i])) for i in bad[:5]])


def _sorted_keys(rng, n, nparts, plen=None):
    """partition keys (runs of plen rows, or random) and order keys with ties"""
    if plen:
        p = np.arange(n) // plen
    else:
        p = np.sort(rng.integers(0, max(nparts, 1), n))
    o = np.zeros(n, dtype=np.int64)
    for g in np.unique(p):
        idx = np.nonzero(p == g)[0]
        o[idx] = np.sort(rng.integers(0, 6, len(idx)))
    return p.astype(np.int64), o


def _nulls(rng, n, density):
    return rng.random(n) >= density


def _check_frames(m, p, o, vcol, valid, frames, part_by=(0,), order=((1, 1, 1),), frames_of=None):
    """every (frame, kind, n, ignore) over column 2 of a table (p, o, v) against the oracle"""
    t = m.Table.from_columns([m.Column.from_numpy(p.astype(np.int32)), m.Column.from_numpy(o), vcol])
    funcs, keys = [], []
    for fr in frames:
        for kind, k in KINDS:
            for ign in (False, True):
                funcs.append(_fn(m, kind, k, 2, fr, ign))
                keys.append((fr, kind, k, ign))
    out = m.window(t, list(part_by), list(order), funcs)
    pk, ok = [(int(x),) for x in p], [(int(x),) for x in o]
    cache = {}
    for j, (fr, kind, k, ign) in enumerate(keys):
        ck = (fr.type, fr.lower, fr.upper)
        if ck not in cache:
            cache[ck] = frames_of(fr) if frames_of else V.frames(pk, ok, fr.type, fr.lower, fr.upper)
        src = V.source_rows(cache[ck], kind, list(valid), k, ign)
        _assert_copied(out.column(3 + j), vcol, src, (ck, kind, k, ign))
    return out


@pytest.mark.parametrize("density", [0.0, 0.1, 0.95, 1.0])
@pytest.mark.parametrize("n,nparts,plen", [(1, 1, None), (31, 2, None), (32, 1, 32), (33, 3, None), (TILE - 1, 7, None), (TILE, 1, None),
                                           (TILE + 1, 3, None), (3 * TILE + 5, 0, 64), (4 * TILE, 0, 1024), (2 * TILE, 0, 32)])
def test_every_frame_and_null_density(b2, n, nparts, plen, density):
    m = b2
    rng = np.random.default_rng(n * 7 + int(density * 100))
    p, o = _sorted_keys(rng, n, nparts, plen)
    valid = _nulls(rng, n, density)
    v = rng.integers(-2 ** 62, 2 ** 62, n)
    vcol = m.Column.from_numpy(v, m.INT64, valid)
    _check_frames(m, p, o, vcol, valid, [m.Frame(ft, lo, up) for ft, lo, up in FRAMES])


def _typed(m, rng, name, n, valid):
    """a value column of type `name` with its edge values, NULL where not valid"""
    dt = getattr(m, name)
    if name == "STRING":
        pool = ["", "a", "bb", "été", "s" * 40]
        vals = [pool[int(i)] if ok else None for i, ok in zip(rng.integers(0, len(pool), n), valid)]
        return m.Column.from_strings(vals)
    if name == "BOOL8":
        return m.Column.from_numpy(rng.integers(0, 2, n).astype(np.int8), m.BOOL8, valid)
    if name in ("FLOAT32", "FLOAT64"):
        nan = _f32_nan if name == "FLOAT32" else _f64_nan
        pool = [nan(0), nan(5), nan(123), -0.0, 0.0, float("inf"), -float("inf"), 1.5, -2.25]
        arr = np.array([pool[int(i)] for i in rng.integers(0, len(pool), n)], dtype=np.float32 if name == "FLOAT32" else np.float64)
        return m.Column.from_numpy(arr, dt, valid)
    if name.startswith("DECIMAL"):
        big = {"DECIMAL32": 10 ** 9 - 1, "DECIMAL64": 10 ** 18 - 1, "DECIMAL128": 10 ** 38 - 1}[name]
        pool = [big, -big, 0, 1, -1, 12345]
        vals = [pool[int(i)] for i in rng.integers(0, len(pool), n)]
        return _column(m, dt, [x if ok else None for x, ok in zip(vals, valid)], True, 2)
    bits = {"INT8": 8, "INT16": 16, "INT32": 32, "INT64": 64, "DATE32": 32, "TIMESTAMP_US": 64}[name]
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    vals = [int(x) for x in rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)]
    return _column(m, dt, [x if ok else None for x, ok in zip(vals, valid)], True)


TYPES = ["BOOL8", "INT8", "INT16", "INT32", "INT64", "DATE32", "TIMESTAMP_US", "FLOAT32", "FLOAT64", "DECIMAL32", "DECIMAL64",
         "DECIMAL128", "STRING"]


@pytest.mark.parametrize("name", TYPES)
def test_every_value_type(b2, name):
    m = b2
    rng = np.random.default_rng(len(name))
    n = TILE + 37
    p, o = _sorted_keys(rng, n, 9)
    valid = _nulls(rng, n, 0.1)
    vcol = _typed(m, rng, name, n, valid)
    frames = [m.rows(None, 0), m.range_running(), m.unbounded(), m.rows(-3, 2), m.rows(1, 4), m.rows(None, 2)]
    _check_frames(m, p, o, vcol, valid, frames)


RANGE_KEYS = {"INT64": ([-2 ** 63, 2 ** 63 - 1, 0, 1, 3, 4, 10, -5], 3), "DATE32": ([0, 1, 7, 8, 30, -365], 7),
              "DECIMAL64": ([-(10 ** 18 - 1), 10 ** 18 - 1, 0, 150, 250, 300], 100)}


@pytest.mark.parametrize("otype", sorted(RANGE_KEYS))
@pytest.mark.parametrize("asc,nulls_first", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_range_value_frames(b2, otype, asc, nulls_first):
    m = b2
    rng = np.random.default_rng(len(otype) * 10 + asc * 2 + nulls_first)
    n = 2 * TILE + 11
    pool, k = RANGE_KEYS[otype]
    o = [None if rng.random() < 0.15 else pool[int(i)] for i in rng.integers(0, len(pool), n)]
    p = [int(x) for x in rng.integers(0, 5, n)]
    valid = _nulls(rng, n, 0.3)
    v = rng.integers(-2 ** 62, 2 ** 62, n)
    scale = 2 if otype.startswith("DECIMAL") else 0
    t = m.Table.from_columns([_column(m, m.INT32, p, False), _column(m, getattr(m, otype), o, True, scale), m.Column.from_numpy(v, m.INT64, valid)])
    srt = m.order_by(t, [(0, 1, 1), (1, asc, nulls_first)])
    cols = srt.to_pylists()
    pk, ok = [(x,) for x in cols[0]], [(x,) for x in cols[1]]
    svalid = [x is not None for x in cols[2]]
    frames = [m.range_between(lo, up) for lo, up in [(-k, 0), (-k, k), (0, k), (1, 3), (0, None), (None, k), (-k, None)]]
    funcs, keys = [], []
    for fr in frames:
        for kind, nth in KINDS:
            for ign in (False, True):
                funcs.append(_fn(m, kind, nth, 2, fr, ign))
                keys.append((fr, kind, nth, ign))
    out = m.window(srt, [0], [(1, asc, nulls_first)], funcs)
    cache = {}
    for j, (fr, kind, nth, ign) in enumerate(keys):
        if (fr.lower, fr.upper) not in cache:
            cache[(fr.lower, fr.upper)] = R.frames(pk, ok, fr.lower, fr.upper, bool(asc), bool(nulls_first))
        src = V.source_rows(cache[(fr.lower, fr.upper)], kind, svalid, nth, ign)
        _assert_copied(out.column(3 + j), srt.column(2), src, (fr.lower, fr.upper, kind, nth, ign))


# ---- GpuWindowExec ---------------------------------------------------------------------------------------------------------------
def _exec(m, t, part, order, funcs, cuts):
    from spark_rapids_b200 import execs as E
    ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, t, cuts)), part, order, funcs)
    got, names = _kernels(m, lambda: list(ex))
    return got, names, ex.metrics


def _assert_exec_equals_window(m, t, part, order, funcs, cuts):
    exp = m.window(t, part, order, funcs)
    got, names, mt = _exec(m, t, part, order, funcs, cuts)
    assert mt["numOutputRows"] == t.num_rows
    whole = m.concat(got) if len(got) > 1 else got[0]
    for c in range(t.num_columns, t.num_columns + len(funcs)):
        ev, eok = exp.column(c).to_numpy()
        gv, gok = whole.column(c).to_numpy()
        assert np.array_equal(np.asarray(eok, bool), np.asarray(gok, bool)), c
        sel = np.nonzero(np.asarray(eok, bool))[0]
        a, b = _raw(ev)[sel], _raw(gv)[sel]
        assert np.array_equal(a, b) if a.dtype != object else list(a) == list(b), c
    return names


def _value_table(m, rng, n, nparts, density):
    p, o = _sorted_keys(rng, n, nparts)
    valid = _nulls(rng, n, density)
    cols = [m.Column.from_numpy(p.astype(np.int32)), m.Column.from_numpy(o), m.Column.from_numpy(rng.integers(-10 ** 6, 10 ** 6, n), m.INT64, valid),
            _typed(m, rng, "STRING", n, valid), _typed(m, rng, "DECIMAL128", n, valid), _typed(m, rng, "FLOAT64", n, valid)]
    return m.Table.from_columns(cols)


def _value_fns(m, fr, with_others):
    out = []
    for c in (2, 3, 4, 5):
        out += [m.first_value(c, fr), m.first_value(c, fr, True), m.last_value(c, fr), m.last_value(c, fr, True),
                m.nth_value(c, 2, fr), m.nth_value(c, 3, fr, True)]
    if with_others:
        out += [m.win_sum(2, fr), m.lag(3, 2), m.row_number()]
    return out


PLANS = {"running": lambda m: m.rows(None, 0), "range_running": lambda m: m.range_running(), "bounded": lambda m: m.rows(-3, 2),
         "bounded_unbounded": lambda m: m.rows(None, 2), "whole": lambda m: m.unbounded(), "range_value": lambda m: m.range_between(-2, 1)}


@pytest.mark.parametrize("plan", sorted(PLANS))
@pytest.mark.parametrize("with_others", [False, True])
@pytest.mark.parametrize("nbatches", [1, 2, 7])
def test_exec_equals_one_batch(b2, plan, with_others, nbatches):
    m = b2
    rng = np.random.default_rng(nbatches * 31 + len(plan) + with_others)
    n = 2 * TILE + 77
    t = _value_table(m, rng, n, 6, 0.6)
    pvals = t.column(0).to_numpy()[0]
    starts = [int(i) for i in np.nonzero(np.diff(pvals))[0] + 1]
    if nbatches == 1:
        cuts = []
    elif nbatches == 2:
        cuts = [starts[0] if starts else n // 2]   # at a partition start
    else:
        mid = starts[len(starts) // 2] if starts else n // 2
        cuts = sorted({int(rng.integers(1, n - 1)), mid, mid + 1, mid + 2, n // 3, n // 3 + 1})[:6]   # one-row batches
    order = [(1, 1, 1)]
    _assert_exec_equals_window(m, t, [0], order, _value_fns(m, PLANS[plan](m), with_others), cuts)


@pytest.mark.parametrize("frame", ["running", "bounded_unbounded"])
def test_forward_fill_across_batches(b2, frame):
    """partition 0: one non-NULL value in the first of 6 batches; partition 1: its first batches all NULL, then values; the n-th
    counted row of NTH_VALUE three batches back; STRING and DECIMAL128 carried values"""
    m = b2
    bl = 50
    n0, n1 = 6 * bl, 5 * bl
    n = n0 + n1
    p = np.array([0] * n0 + [1] * n1, dtype=np.int32)
    o = np.arange(n, dtype=np.int64)
    valid = np.zeros(n, bool)
    valid[[3, 7, 9]] = True                       # partition 0: three values, all in batch 0
    valid[n0 + 3 * bl + 5:] = True                 # partition 1: NULL for three batches
    rng = np.random.default_rng(4)
    t = m.Table.from_columns([m.Column.from_numpy(p), m.Column.from_numpy(o), m.Column.from_numpy(rng.integers(-99, 99, n), m.INT64, valid),
                              _typed(m, rng, "STRING", n, valid), _typed(m, rng, "DECIMAL128", n, valid), _typed(m, rng, "FLOAT64", n, valid)])
    fr = PLANS[frame](m)
    funcs = []
    for c in (2, 3, 4, 5):
        funcs += [m.last_value(c, fr, True), m.first_value(c, fr, True), m.nth_value(c, 3, fr, True), m.nth_value(c, 2, fr), m.first_value(c, fr)]
    cuts = [bl * k for k in range(1, 11)]
    _assert_exec_equals_window(m, t, [0], [(1, 1, 1)], funcs, cuts)
    # and against the oracle directly
    out = m.window(t, [0], [(1, 1, 1)], funcs)
    pk, ok = [(int(x),) for x in p], [(int(x),) for x in o]
    frs = V.frames(pk, ok, W.ROWS, fr.lower, fr.upper)
    for j, (kind, k, ign) in enumerate([(V.LAST, 1, True), (V.FIRST, 1, True), (V.NTH_VALUE, 3, True), (V.NTH_VALUE, 2, False), (V.FIRST, 1, False)]):
        for ci, c in enumerate((2, 3, 4, 5)):
            _assert_copied(out.column(6 + ci * 5 + j), t.column(c), V.source_rows(frs, kind, list(valid), k, ign), (kind, k, ign, c))


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


@pytest.mark.parametrize("plan", ["running", "bounded"])
def test_split_under_an_allocation_limit(b2, limits, plan):
    """as test_window_gpu's and test_window_bounded_stream_gpu's split tests, with a forward fill beside (running) or in place of
    LAG (bounded): under 54 B per row the batch is halved, and the halves, continued through the carry, equal the whole"""
    m = b2
    from spark_rapids_b200 import execs as E
    n = 1 << 21
    rng = np.random.default_rng(17)
    if plan == "running":
        key = np.sort(rng.integers(0, 5000, n)).astype(np.int64)
        funcs = [m.row_number(), m.win_sum(1, m.rows(None, 0)), m.last_value(1, m.rows(None, 0), True)]
        part, order = [0], [(0, 1, 1)]
    else:
        key = np.arange(n, dtype=np.int64)
        funcs = [m.row_number(), m.last_value(1, m.rows(None, 2), True), m.win_sum(1, m.rows(-3, 3))]
        part, order = [], [(0, 1, 1)]
    val = rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64)
    t = m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(val, m.INT64, rng.random(n) < 0.1)])
    ref = m.window(t, part, order, funcs)
    exp = [ref.column(2 + k).to_numpy() for k in range(len(funcs))]
    del ref
    src = E.GpuBatchSource([t])
    del t
    gc.collect()
    m.sync()
    s0 = m.memory_stats()
    m.set_alloc_limit(m.device_bytes_in_use() + 54 * n)
    ex = E.GpuWindowExec(src, part, order, funcs)
    del src
    got = [[] for _ in funcs]
    nout = 0
    while True:
        b = ex.next()
        if b is None:
            break
        for k in range(len(funcs)):
            got[k].append(b.column(2 + k).to_numpy())
        nout += 1
        del b
    m.set_alloc_limit(0)
    s1 = m.memory_stats()
    assert s1["splits"] > s0["splits"] and nout >= 2, (s0, s1, nout)
    for k in range(len(funcs)):
        vals, ok = np.concatenate([g[0] for g in got[k]]), np.concatenate([g[1] for g in got[k]])
        assert np.array_equal(ok, exp[k][1]) and np.array_equal(vals[ok], exp[k][0][ok]), k


def test_argument_errors(b2):
    m = b2
    t = m.Table.from_columns([_column(m, m.INT32, [1, 1], False), _column(m, m.INT64, [1, 2], False), m.Column.from_strings(["a", "b"]),
                              _column(m, m.FLOAT64, [1.0, 2.0], False)])
    sum_ign = m.WindowFunc(m.WIN_SUM, 1, m.rows(None, 0), ignore_nulls=True)
    lag_ign = m.WindowFunc(m.WIN_LAG, 1, offset=1, ignore_nulls=True)
    cases = [
        ([(1, 1, 1)], m.nth_value(2, 0, m.rows(None, 0)), INVALID),
        ([(1, 1, 1)], m.nth_value(2, -3, m.rows(None, 0)), INVALID),
        ([(1, 1, 1)], sum_ign, INVALID),
        ([(1, 1, 1)], m.WindowFunc(m.WIN_COUNT_ALL, 0, m.unbounded(), ignore_nulls=True), INVALID),
        ([(1, 1, 1)], lag_ign, UNSUPPORTED),
        ([(1, 1, 1)], m.first_value(2, m.rows(2, 1)), INVALID),                       # lower > upper
        ([(1, 1, 1)], m.last_value(2, m.Frame(m.FRAME_RANGE, -1, 0)), UNSUPPORTED),   # RANGE with a value offset
        ([], m.first_value(2, m.range_between(-1, 0)), INVALID),                     # no ORDER BY
        ([(3, 1, 1)], m.last_value(2, m.range_between(-1, 0)), UNSUPPORTED),         # float ORDER BY
        ([(2, 1, 1)], m.last_value(1, m.range_between(-1, 0)), INVALID),             # STRING ORDER BY
        ([(1, 1, 1)], m.first_value(9, m.unbounded()), INVALID),                     # column out of range
    ]
    for order, f, code in cases:
        with pytest.raises(m.B2Error) as ei:
            m.window(t, [0], order, [f])
        assert ei.value.code == code, (f.kind, ei.value)
    # a STRING result, "" apart from NULL, and no ORDER BY for the whole partition
    t2 = m.Table.from_columns([_column(m, m.INT32, [1, 1, 1], False), m.Column.from_strings([None, "", "x"])])
    out = m.window(t2, [0], [], [m.first_value(1, m.unbounded()), m.first_value(1, m.unbounded(), True), m.last_value(1, m.unbounded())])
    assert [out.column(c).to_pylist() for c in (2, 3, 4)] == [[None] * 3, [""] * 3, ["x"] * 3]
