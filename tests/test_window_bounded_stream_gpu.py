"""GpuWindowExec streaming bounded plans (ranking, LEAD / LAG, ROWS frames with a finite upper bound) batch by batch with context
and look-ahead rows, against b2_window over the concatenated input: exact, float sums included (every partial sum of these
inputs is exact in double)."""
import gc

import numpy as np
import pytest

from tests.test_window_gpu import TILE, VALUE_TYPES, _batches, _kernels, _matrix_case, _same, _sorted_input, _table

pytestmark = pytest.mark.gpu

INPUT_COLS = 7   # _table: p, o, i64, f64, d38, d18, str


def _lag_lead_plan(m):
    out = [m.row_number(), m.rank(), m.dense_rank()]
    for off in (1, 2, 7):
        out += [m.lag(2, off), m.lead(2, off, default=-7), m.lag(3, off, default=2.5, dtype=m.FLOAT64), m.lead(6, off), m.lag(4, off)]
    return out


BOUNDED_FRAMES = [(-6, 0), (-2, 2), (0, 3), (-5, -2), (2, 5), (None, 3), (None, -2)]


def _frames_plan(m):
    out = [m.row_number(), m.rank(), m.dense_rank(), m.win_sum(2, m.rows(None, 0)), m.win_sum(3, m.rows(None, 0))]
    for lo, up in BOUNDED_FRAMES:
        fr = m.rows(lo, up)
        out += [m.win_sum(2, fr), m.win_sum(3, fr), m.win_sum(5, fr, m.DECIMAL128, 28), m.win_count(2, fr), m.win_count_all(fr),
                m.win_min(2, fr), m.win_max(3, fr)]
    return out


PLANS = {"lag_lead": _lag_lead_plan, "frames": _frames_plan}


def _cuts(rng, n, nbatches):
    """nbatches - 1 cut points with repeats (empty batches) and a 1-row batch"""
    if nbatches == 1:
        return []
    cuts = sorted(int(x) for x in rng.integers(1, n - 1, nbatches - 1))
    cuts[len(cuts) // 2] = min(cuts[len(cuts) // 2], n - 2)
    extra = [cuts[0], cuts[len(cuts) // 2] + 1]   # an empty batch and a 1-row batch
    return sorted(cuts + extra)


def _stream(m, t, part, order, funcs, cuts):
    """GpuWindowExec over the cut batches: (output batches, kernel names, metrics)"""
    from spark_rapids_b200 import execs as E
    ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, t, cuts)), part, order, funcs)
    got, names = _kernels(m, lambda: list(ex))
    return got, names, ex.metrics


def _assert_same_columns(exp, got_batches, first, nfuncs):
    ecols = exp.to_pylists()
    gcols = [[] for _ in range(first + nfuncs)]
    for b in got_batches:
        for c, v in enumerate(b.to_pylists()):
            gcols[c] += v
    for c in range(first + nfuncs):
        assert _same(gcols[c], ecols[c]), (c, [(i, g, e) for i, (g, e) in enumerate(zip(gcols[c], ecols[c])) if not _same([g], [e])][:5])


def _nonempty(cuts, n):
    return len([1 for a, b in zip([0] + list(cuts), list(cuts) + [n]) if b > a])


@pytest.mark.parametrize("plan", sorted(PLANS))
@pytest.mark.parametrize("parts", ["none", "many", "one"])
@pytest.mark.parametrize("nbatches", [1, 2, 7, 40])
def test_stream_equals_one_batch(b2, plan, parts, nbatches):
    m = b2
    rng = np.random.default_rng(100 * nbatches + 10 * sorted(PLANS).index(plan) + ["none", "many", "one"].index(parts))
    n = 3 * TILE + 17
    p, o, vals = _sorted_input(rng, n, {"none": 1, "many": 60, "one": 1}[parts])
    t = _table(m, p, o, vals)
    part = [] if parts == "none" else [0]
    order = [(0, 1, 1), (1, 1, 1)] if parts == "none" else [(1, 1, 1)]
    funcs = PLANS[plan](m)
    exp = m.window(t, part, order, funcs)
    cuts = _cuts(rng, n, nbatches)
    got, names, mt = _stream(m, t, part, order, funcs, cuts)
    _assert_same_columns(exp, got, INPUT_COLS, len(funcs))
    assert "window_last_start_kernel" not in names and "window_finish_kernel" in names
    assert mt["numOutputRows"] == n and mt["numOutputBatches"] == _nonempty(cuts, n) == len(got)


@pytest.mark.parametrize("shift", [0, 1, 7, 8, 9])
def test_partition_starts_at_and_before_a_batch_edge(b2, shift):
    """P = 7 (LAG 7, ROWS -6..0 and -5..-2): a partition starts `shift` rows before each batch edge"""
    m = b2
    rng = np.random.default_rng(50 + shift)
    edges = [500, 1100, 1700, 2300]
    n = 2900
    starts = [0] + [e - shift for e in edges]
    p = [sum(1 for s in starts if s <= i) for i in range(n)]
    _, _, vals = _sorted_input(rng, n, 1)
    o = [i % 5 for i in range(n)]
    o = [x for _, x in sorted(zip(p, o))]
    t = _table(m, p, o, vals)
    funcs = [m.lag(2, 7, default=3), m.lead(2, 2), m.win_sum(2, m.rows(-6, 0)), m.win_min(2, m.rows(-5, -2)), m.win_sum(5, m.rows(None, -2), m.DECIMAL128, 28),
             m.win_count(2, m.rows(-6, 2)), m.row_number(), m.rank(), m.win_sum(3, m.rows(None, 0))]
    exp = m.window(t, [0], [(1, 1, 1)], funcs)
    got, names, mt = _stream(m, t, [0], [(1, 1, 1)], funcs, edges)
    _assert_same_columns(exp, got, INPUT_COLS, len(funcs))
    assert mt["numOutputBatches"] == len(edges) + 1


@pytest.mark.parametrize("parts", ["none", "one"])
def test_frames_wider_than_a_batch_and_than_the_input(b2, parts):
    """ROWS -1000..1000 and LAG / LEAD 60 over 40 batches of 1 to 50 rows: the context and look-ahead span many batches"""
    m = b2
    rng = np.random.default_rng(61)
    sizes = [int(x) for x in rng.integers(1, 51, 40)]
    n = sum(sizes)
    p, o, vals = _sorted_input(rng, n, 1)
    t = _table(m, p, o, vals)
    fr = m.rows(-1000, 1000)
    funcs = [m.win_sum(2, fr), m.win_sum(3, fr), m.win_count(2, fr), m.win_min(2, fr), m.win_max(3, fr), m.win_sum(5, fr, m.DECIMAL128, 28),
             m.lag(6, 60), m.lead(2, 60, default=1), m.win_sum(2, m.rows(-30, -20)), m.row_number()]
    part = [] if parts == "none" else [0]
    exp = m.window(t, part, [(1, 1, 1)], funcs)
    cuts = list(np.cumsum(sizes)[:-1])
    got, names, mt = _stream(m, t, part, [(1, 1, 1)], funcs, cuts)
    _assert_same_columns(exp, got, INPUT_COLS, len(funcs))
    assert mt["numOutputBatches"] == 40 and "window_last_start_kernel" not in names


@pytest.mark.parametrize("nullable", [True, False])
def test_lead_lag_over_every_type(b2, nullable):
    m = b2
    n = 2 * TILE + 37
    srt, part_cols, order, nkeys = _matrix_case(m, 70, ["INT32"], [("INT64", 1, 1)], nullable, n)
    funcs = []
    for j, name in enumerate(VALUE_TYPES):
        c = nkeys + j
        vt_float = name.startswith("FLOAT")
        default = None if name == "STRING" else 1.5 if vt_float else 2
        funcs += [m.lag(c, 1, default=default, dtype=getattr(m, name) if vt_float else None), m.lead(c, 3), m.lag(c, 9)]
    exp = m.window(srt, part_cols, order, funcs)
    cuts = sorted(int(x) for x in np.random.default_rng(3).integers(0, n, 8))
    got, names, mt = _stream(m, srt, part_cols, order, funcs, cuts)
    _assert_same_columns(exp, got, srt.num_columns, len(funcs))
    assert "window_last_start_kernel" not in names


def test_decimal_sums_overflow_to_null_across_chunk_edges(b2):
    """a bounded DECIMAL(38) SUM whose frame total overflows is NULL, and is valid again once the frame has passed the large
    values; a running SUM that overflows stays NULL for the rest of the partition, across every batch edge after it"""
    m = b2
    from spark_rapids_b200 import execs as E
    big = 10 ** 38 - 1
    n = 2 * TILE + 10
    d = [1] * n
    d[3], d[4], d[TILE + 3] = big - 5, big, -(n + 10)
    t = m.Table.from_columns([m.Column.from_numpy(np.zeros(n, np.int32)), m.Column.from_numpy(np.arange(n, dtype=np.int64)),
                              m.Column.from_numpy(np.array(d, dtype=object), m.DECIMAL128, None, 0)])
    funcs = [m.win_sum(2, m.rows(None, 0), m.DECIMAL128, 38), m.win_sum(2, m.rows(-1, 1), m.DECIMAL128, 38), m.lag(2, 1)]
    exp = m.window(t, [0], [(1, 1, 1)], funcs)
    cuts = [2, 5, 100, TILE, TILE + 4, 2 * TILE]
    ex = E.GpuWindowExec(E.GpuBatchSource(_batches(m, t, cuts)), [0], [(1, 1, 1)], funcs)
    got = list(ex)
    _assert_same_columns(exp, got, 3, len(funcs))
    run = [v for b in got for v in b.column(3).to_pylist()]
    assert run[3] == big - 2 and all(v is None for v in run[4:])
    mov = [v for b in got for v in b.column(4).to_pylist()]
    assert mov[2] == big - 3 and mov[3] is None and mov[5] is None and mov[6] == 3


def test_pass_through_columns_are_the_input_batches(b2):
    """each output batch holds its input batch's own columns (same device buffers), then the function columns"""
    m = b2
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(71)
    n = 3 * TILE
    p, o, vals = _sorted_input(rng, n, 9)
    t = _table(m, p, o, vals)
    cuts = [0, 700, 700, 701, 2000]
    batches = _batches(m, t, cuts)
    ptrs = [[b.column(c).info().data for c in range(INPUT_COLS)] for b in batches if b.num_rows]
    funcs = [m.lag(2, 2), m.win_sum(2, m.rows(-3, 1)), m.row_number()]
    ex = E.GpuWindowExec(E.GpuBatchSource(batches), [0], [(1, 1, 1)], funcs)
    got = list(ex)
    assert len(got) == len(ptrs) == ex.metrics["numOutputBatches"] and ex.metrics["numOutputRows"] == n
    for b, want in zip(got, ptrs):
        assert b.num_columns == INPUT_COLS + len(funcs)
        assert [b.column(c).info().data for c in range(INPUT_COLS)] == want


@pytest.mark.parametrize("extra", ["unbounded_following", "range_running", "range_unbounded"])
def test_a_whole_partition_or_range_function_keeps_the_held_partition_path(b2, extra):
    m = b2
    rng = np.random.default_rng(81)
    n = 2 * TILE + 5
    p, o, vals = _sorted_input(rng, n, 1)
    t = _table(m, p, o, vals)
    base = [m.lag(2, 1), m.win_sum(2, m.rows(-6, 0)), m.row_number()]
    add = {"unbounded_following": m.win_sum(2, m.rows(-2, None)), "range_running": m.win_sum(2, m.range_running()),
           "range_unbounded": m.win_count(2, m.Frame(m.FRAME_RANGE, None, None))}[extra]
    funcs = base + [add]
    exp = m.window(t, [], [(1, 1, 1)], funcs)
    cuts = [300, 900, 1500]
    got, names, mt = _stream(m, t, [], [(1, 1, 1)], funcs, cuts)
    _assert_same_columns(exp, got, INPUT_COLS, len(funcs))
    assert "window_last_start_kernel" in names
    assert len(got) == 1   # no PARTITION BY: the whole input is one held group, as before
    got2, names2, mt2 = _stream(m, t, [], [(1, 1, 1)], base, cuts)
    assert "window_last_start_kernel" not in names2 and len(got2) == 4


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


def _sliding(v, lo, up, fn, fill):
    """fn over v[i + lo .. i + up] clipped to the array, for every i (no PARTITION BY)"""
    n = len(v)
    out = np.full(n, fill, dtype=v.dtype)
    for d in range(lo, up + 1):
        src = np.arange(n) + d
        ok = (src >= 0) & (src < n)
        out[ok] = fn(out[ok], v[src[ok]])
    return out


def test_larger_than_the_allocation_limit_streams(b2, limits):
    """256 MiB of (INT64 order key, INT64 value) from host batches of 8 MiB, no PARTITION BY, under an allocation limit of
    64 MiB above the base.  Before bounded plans streamed, the whole input was one held group, concatenated on the device,
    and this failed with B2_ERR_OOM.  Each output batch is copied to the host, released and checked against numpy."""
    m = b2
    from spark_rapids_b200 import execs as E
    rows, nb = 1 << 19, 32
    n = rows * nb
    rng = np.random.default_rng(91)
    ts = np.arange(n, dtype=np.int64) * 3
    v = rng.integers(-10**9, 10**9, n).astype(np.int64)
    batches = [[(m.INT64, 0, ts[s:s + rows], None), (m.INT64, 0, v[s:s + rows], None)] for s in range(0, n, rows)]
    exp_lag = np.concatenate([[0], v[:-1]])
    exp_lead = np.concatenate([v[2:], [0, 0]])
    exp_sum = _sliding(v, -6, 0, np.add, 0)
    exp_min = _sliding(v, -2, 2, np.minimum, np.iinfo(np.int64).max)
    gc.collect()
    m.sync()
    base = m.device_bytes_in_use()
    m.set_alloc_limit(base + (64 << 20))
    funcs = [m.lag(1, 1), m.lead(1, 2), m.win_sum(1, m.rows(-6, 0)), m.win_min(1, m.rows(-2, 2)), m.row_number()]
    ex = E.GpuWindowExec(E.GpuHostBatchSource(batches), [], [(0, 1, 1)], funcs)
    at, nout = 0, 0
    while True:
        b = ex.next()
        if b is None:
            break
        k = b.num_rows
        cols = [b.column(c).to_numpy() for c in range(7)]
        del b
        sl = slice(at, at + k)
        assert np.array_equal(cols[0][0], ts[sl]) and np.array_equal(cols[1][0], v[sl])
        (lag_v, lag_ok), (lead_v, lead_ok) = cols[2], cols[3]
        idx = np.arange(at, at + k)
        assert np.array_equal(lag_ok, idx >= 1) and np.array_equal(lag_v[lag_ok], exp_lag[sl][lag_ok])
        assert np.array_equal(lead_ok, idx < n - 2) and np.array_equal(lead_v[lead_ok], exp_lead[sl][lead_ok])
        assert np.array_equal(cols[4][0], exp_sum[sl]) and np.array_equal(cols[5][0], exp_min[sl])
        assert np.array_equal(cols[6][0], (idx + 1).astype(np.int32))
        at += k
        nout += 1
    m.set_alloc_limit(0)
    assert at == n and ex.metrics["numOutputRows"] == n and ex.metrics["numOutputBatches"] == nout >= nb
    del ex
    gc.collect()
    m.sync()
    assert m.device_bytes_in_use() <= base


def test_split_and_retry_under_an_allocation_limit(b2, limits):
    """one batch of 2^21 rows needs about 73 B per row at its peak; a half, with both halves' copies, about 45.  Under a limit of
    54 B per row the batch is halved; the halves leave as two output batches and equal the whole"""
    m = b2
    from spark_rapids_b200 import execs as E
    n = 1 << 21
    rng = np.random.default_rng(93)
    key = np.arange(n, dtype=np.int64)
    val = rng.integers(-10**6, 10**6, n).astype(np.int64)
    funcs = [m.row_number(), m.lag(1, 1), m.win_sum(1, m.rows(-3, 3))]
    t = m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(val)])
    ref = m.window(t, [], [(0, 1, 1)], funcs)
    exp = [ref.column(2 + k).to_numpy() for k in range(len(funcs))]
    del ref
    src = E.GpuBatchSource([t])
    del t
    gc.collect()
    m.sync()
    s0 = m.memory_stats()
    m.set_alloc_limit(m.device_bytes_in_use() + 54 * n)
    ex = E.GpuWindowExec(src, [], [(0, 1, 1)], funcs)
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
    assert ex.metrics["numOutputRows"] == n and ex.metrics["numOutputBatches"] == nout


def test_past_2_31_rows(b2):
    """2^31 + 2^20 rows of (INT32 order key = position, INT32 v = position mod 1000) in host batches of 2^27 rows, no PARTITION
    BY: LAG(v, 1) and ROWS -3..0 COUNT(*) and SUM(v), checked on the device batch by batch against the closed form.  Before
    bounded plans streamed, the whole input was one group and this failed with B2_ERR_SIZE_OVERFLOW."""
    from spark_rapids_b200 import execs as E
    m = b2
    n, rows = (1 << 31) + (1 << 20), 1 << 27
    pos = np.arange(n, dtype=np.uint32).view(np.int32)
    v = np.tile(np.arange(1000, dtype=np.int32), n // 1000 + 1)[:n]
    batches = [[(m.INT32, 0, pos[s:s + rows], None), (m.INT32, 0, v[s:s + rows], None)] for s in range(0, n, rows)]
    funcs = [m.lag(1, 1), m.win_count_all(m.rows(-3, 0)), m.win_sum(1, m.rows(-3, 0))]
    cv = m.col(1, m.INT32, nullable=False)
    lag, cnt, sm = m.col(2, m.INT32), m.col(3, m.INT64), m.col(4, m.INT64)
    v64 = cv.cast(m.INT64)
    exp_sum = v64
    for d in range(1, 4):
        exp_sum = exp_sum + (v64 + m.lit(1000 - d, m.INT64)) % m.lit(1000, m.INT64)
    bad = (lag.is_null() | (lag != (cv + m.lit(999, m.INT32)) % m.lit(1000, m.INT32)) | (cnt != m.lit(4, m.INT64)) | sm.is_null()
           | (sm != exp_sum))
    prog = m.Program([bad])
    ex = E.GpuWindowExec(E.GpuHostBatchSource(batches), [], [(0, 1, 1)], funcs)
    total, nout, mismatches = 0, 0, 0
    for t in ex:
        assert t.num_rows < 2**31
        if nout == 0:
            head = m.slice_table(t, 0, 4).to_rows()
            assert [tuple(r[2:]) for r in head] == [(None, 1, 0), (0, 2, 1), (1, 3, 3), (2, 4, 6)]
        mismatches += m.filter_count(prog, t)
        total += t.num_rows
        nout += 1
        del t
    assert mismatches == 3   # rows 0..2 of the input, checked above
    assert total == n and nout == len(batches) and ex.metrics["numOutputRows"] == n
