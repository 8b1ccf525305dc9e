"""The merge-path merge of sorted runs (b2_merge_sorted) and the out-of-core GpuSortExec (GpuOutOfCoreSortIterator), checked
row for row against a stable sort: oracle.spark_relational.sort_order up to ~20 K rows, numpy's stable sorts above that."""
import gc

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from tests import datagen as G

pytestmark = pytest.mark.gpu

ORDERS = [(1, 1), (1, 0), (0, 1), (0, 0)]   # (ascending, nulls_first)
KEY_TYPES = [(O.INT8, 0, 0), (O.INT16, 0, 0), (O.INT32, 0, 0), (O.INT64, 0, 0), (O.DATE32, 0, 0), (O.TIMESTAMP_US, 0, 0),
             (O.FLOAT32, 0, 0), (O.FLOAT64, 0, 0), (O.DECIMAL32, 9, 2), (O.DECIMAL64, 18, 2), (O.DECIMAL128, 38, 2), (O.STRING, 0, 0)]


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)
    b2.semaphore_init(0)


def _strings(rng, n, maxlen):
    """empty strings, shared prefixes, non-ASCII bytes; the longest value is exactly maxlen bytes when n > 0"""
    stems = [b"", b"a", b"ab", b"abc", b"abd", "été".encode(), b"\xff", b"zz", b"a\x00"]
    out = []
    for i in range(n):
        s = stems[rng.integers(0, len(stems))]
        s = (s + bytes(rng.integers(97, 100, rng.integers(0, 4)).astype(np.uint8)))[:maxlen]
        out.append(s)
    if n:
        out[rng.integers(0, n)] = (b"ab" * maxlen)[:maxlen]
    return np.array(out, dtype=object)


def _key(rng, typ, n, nullable, maxlen=8):
    dt = typ[0]
    if dt == O.STRING:
        c = O.OCol(_strings(rng, n, maxlen), np.ones(n, bool), typ)
    elif dt == O.TIMESTAMP_US:
        v = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True)
        v[: min(n, 3)] = [-2**63, 2**63 - 1, 0][: min(n, 3)]
        c = O.OCol(v, np.ones(n, bool), typ)
    elif O.is_decimal(dt):
        lim = 10 ** typ[1] - 1
        v = np.array([int(x) for x in rng.integers(-5, 5, n)], dtype=object)
        ext = [lim, -lim, 0, lim - 1, -lim + 1]
        for i in range(min(n, len(ext))):
            v[rng.integers(0, n)] = ext[i]
        c = O.OCol(v, np.ones(n, bool), typ)
    else:
        c = G.gen_column(rng, typ, n, null_frac=0.0, small=n > 0 and rng.random() < 0.5)
    if nullable and n:
        c = O.OCol(c.values, rng.random(n) >= 0.2, typ)
    return c


def _payload(start, n):
    return O.OCol(np.arange(start, start + n, dtype=np.int32), np.ones(n, bool), (O.INT32, 0, 0))


def _cat(batches):
    ncol = len(batches[0])
    return [O.OCol(np.concatenate([b[c].values for b in batches]), np.concatenate([b[c].valid for b in batches]), batches[0][c].typ)
            for c in range(ncol)]


def _sorted_run(cols, keys):
    return R.take(cols, R.sort_order(cols, keys))


def _assert_table(t, cols):
    assert t.num_rows == len(cols[0].values)
    for i, oc in enumerate(cols):
        vals, valid = t.column(i).to_numpy()
        assert np.array_equal(valid, oc.valid), "column %d validity" % i
        got, exp = list(vals[valid]), list(oc.values[oc.valid])
        if oc.typ[0] in (O.FLOAT32, O.FLOAT64):
            g, e = np.asarray(got, dtype=np.float64), np.asarray(exp, dtype=np.float64)
            assert np.array_equal(np.isnan(g), np.isnan(e)) and np.array_equal(g[~np.isnan(g)], e[~np.isnan(e)]), "column %d" % i
        else:
            assert [int(x) if not isinstance(x, bytes) else x for x in got] == [int(x) if not isinstance(x, bytes) else x for x in exp], \
                "column %d" % i


def _table_bytes(t):
    """device bytes as the spill store counts them: data + validity + offsets"""
    b = 0
    for i in range(t.num_columns):
        ci = t.column(i).info()
        n = ci.size
        b += ci.data_bytes + ((n + 1) * 4 if ci.dtype == O.STRING else 0) + ((n + 511) // 512 * 64 if ci.validity else 0)
    return b


# ---- 1. the merge kernel ------------------------------------------------------------------------------------------------------
def _merge_case(b2, rng, typ, k, asc, nf):
    sizes = [[0, 1, 37, 700, 5, 1200, 1, 0, 300][(r * 7 + k) % 9] for r in range(k)]
    maxlens = [3 if r % 2 else 200 for r in range(k)]
    keys = [(0, asc, nf)]
    runs, base = [], 0
    for r in range(k):
        cols = [_key(rng, typ, sizes[r], nullable=r % 2 == 1, maxlen=maxlens[r]), _payload(base, sizes[r])]
        base += sizes[r]
        runs.append(_sorted_run(cols, keys))
    got = b2.merge_sorted([G.to_b2_table(b2, r) for r in runs], keys)
    allc = _cat(runs)
    _assert_table(got, R.take(allc, R.sort_order(allc, keys)))


@pytest.mark.parametrize("typ", KEY_TYPES, ids=lambda t: str(t[0]))
@pytest.mark.parametrize("k", [1, 2, 3, 17])
def test_merge_matches_stable_sort(b2, typ, k):
    rng = np.random.default_rng(1000 * typ[0] + k)
    for asc, nf in ORDERS:
        _merge_case(b2, rng, typ, k, asc, nf)


def test_merge_four_keys_with_ties(b2):
    rng = np.random.default_rng(5)
    keys = [(0, 1, 0), (1, 0, 1), (2, 1, 1), (3, 0, 0)]
    runs, base = [], 0
    for r, n in enumerate([400, 0, 1, 900, 250]):
        cols = [O.OCol(rng.integers(0, 3, n).astype(np.int32), rng.random(n) >= 0.1 * (r % 2), (O.INT32, 0, 0)),
                O.OCol(np.array([[b"", b"x", "ü".encode()][i] for i in rng.integers(0, 3, n)], dtype=object), np.ones(n, bool), (O.STRING, 0, 0)),
                O.OCol(rng.integers(0, 2, n).astype(np.float64) * np.where(rng.random(n) < 0.5, -0.0, 1.0), np.ones(n, bool), (O.FLOAT64, 0, 0)),
                O.OCol(np.array([int(x) for x in rng.integers(-2, 2, n)], dtype=object), rng.random(n) >= 0.1, (O.DECIMAL128, 38, 0)),
                _payload(base, n)]
        base += n
        runs.append(_sorted_run(cols, keys))
    got = b2.merge_sorted([G.to_b2_table(b2, r) for r in runs], keys)
    allc = _cat(runs)
    _assert_table(got, R.take(allc, R.sort_order(allc, keys)))


def test_merge_all_equal_keeps_run_order(b2):
    n = 5000
    a = [O.OCol(np.full(n, 7, np.int64), np.ones(n, bool), (O.INT64, 0, 0)), _payload(0, n)]
    b = [O.OCol(np.full(n, 7, np.int64), np.ones(n, bool), (O.INT64, 0, 0)), _payload(n, n)]
    got = b2.merge_sorted([G.to_b2_table(b2, a), G.to_b2_table(b2, b)], [(0, 1, 1)])
    assert np.array_equal(got.column(1).to_numpy()[0], np.arange(2 * n, dtype=np.int32))


def test_merge_two_runs_of_20m_rows(b2):
    """tile and partition boundaries fall inside long runs of equal keys; only the merge kernels run"""
    rng = np.random.default_rng(9)
    n = 20_000_000
    ka, kb = np.sort(rng.integers(0, 1000, n)).astype(np.int64), np.sort(rng.integers(0, 1000, n)).astype(np.int64)
    ta = b2.Table.from_columns([b2.Column.from_numpy(ka), b2.Column.from_numpy(np.arange(n, dtype=np.int64))])
    tb = b2.Table.from_columns([b2.Column.from_numpy(kb), b2.Column.from_numpy(np.arange(n, 2 * n, dtype=np.int64))])
    b2.sync()
    b2.profile_enable(True)
    try:
        got = b2.merge_sorted([ta, tb], [(0, 1, 1)])
        b2.sync()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    assert {"merge_path_partition_kernel", "merge_path_kernel"} <= names, names
    assert not any(x.startswith("radix_") or x == "small_sort_kernel" for x in names), names
    keys = np.concatenate([ka, kb])
    perm = np.argsort(keys, kind="stable")
    assert np.array_equal(got.column(0).to_numpy()[0], keys[perm])
    assert np.array_equal(got.column(1).to_numpy()[0], perm)


# ---- 2. the out-of-core GpuSortExec -------------------------------------------------------------------------------------------
def _run_ooc(b2, batches, keys, target, check_rows=True):
    from spark_rapids_b200 import execs as E
    b2.sync()
    base = b2.device_bytes_in_use()
    node = E.GpuSortExec(keys, E.GpuBatchSource([G.to_b2_table(b2, b) for b in batches]), target_bytes=target)
    outs = list(node)
    eff = max(target, 16 << 10)
    for t in outs:
        assert t.num_rows >= 1
        assert t.num_rows == 1 or _table_bytes(t) <= eff, (_table_bytes(t), eff)
        del t
    met = node.metrics
    assert met["numOutputBatches"] == len(outs) and met["numOutputRows"] == sum(t.num_rows for t in outs)
    nonempty = [b for b in batches if len(b[0].values)]
    if check_rows and nonempty:
        allc = _cat(nonempty)
        exp = R.take(allc, R.sort_order(allc, keys))
        _assert_table(b2.concat(outs) if len(outs) > 1 else outs[0], exp)
    n = len(outs)
    del outs, node
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base
    return n


def _batches(rng, typ, nb, rows, nullable_every=2, maxlen=8):
    out, base = [], 0
    for b in range(nb):
        n = rows if not callable(rows) else rows(b)
        out.append([_key(rng, typ, n, nullable=b % nullable_every == 1, maxlen=maxlen if b % 2 else 3), _payload(base, n)])
        base += n
    return out


@pytest.mark.parametrize("target", [16 << 10, 100 << 10, 1 << 20, 4 << 20])
@pytest.mark.parametrize("nb", [1, 3, 40])
def test_out_of_core_sort_int_keys(b2, target, nb):
    rng = np.random.default_rng(nb * 31 + target % 97)
    batches = _batches(rng, (O.INT32, 0, 0), nb, lambda b: int(rng.integers(1, 1200)))
    n = _run_ooc(b2, batches, [(0, 1, 1)], target)
    total = sum(len(b[0].values) for b in batches) * 8 + 1024
    if total > 2 * target:
        assert n > 1


@pytest.mark.parametrize("typ", KEY_TYPES, ids=lambda t: str(t[0]))
def test_out_of_core_sort_key_types(b2, typ):
    rng = np.random.default_rng(77 + typ[0])
    for asc, nf in ORDERS:
        batches = _batches(rng, typ, 6, lambda b: [0, 1, 300, 500, 250, 40][b], maxlen=200)
        assert _run_ooc(b2, batches, [(0, asc, nf)], 16 << 10) >= 1


def test_out_of_core_sort_all_keys_equal(b2):
    batches = [[O.OCol(np.zeros(2000, np.int64), np.ones(2000, bool), (O.INT64, 0, 0)), _payload(2000 * b, 2000)] for b in range(12)]
    assert _run_ooc(b2, batches, [(0, 1, 1)], 16 << 10) > 1


@pytest.mark.parametrize("direction", ["sorted", "reverse"])
def test_out_of_core_sort_presorted(b2, direction):
    n, nb = 3000, 10
    vals = np.arange(n * nb, dtype=np.int64)
    if direction == "reverse":
        vals = vals[::-1].copy()
    batches = [[O.OCol(vals[b * n:(b + 1) * n], np.ones(n, bool), (O.INT64, 0, 0)), _payload(b * n, n)] for b in range(nb)]
    assert _run_ooc(b2, batches, [(0, 1, 1)], 32 << 10) > 1


def test_out_of_core_sort_wide_rows(b2):
    """string keys, and rows (a wide payload string) larger than target/8 and than the target itself"""
    rng = np.random.default_rng(3)
    batches, base = [], 0
    for b in range(5):
        n = 60
        key = O.OCol(_strings(rng, n, 40), np.ones(n, bool), (O.STRING, 0, 0))
        wide = O.OCol(np.array([b"w" * int(rng.choice([10, 3000, 20000])) for _ in range(n)], dtype=object), np.ones(n, bool), (O.STRING, 0, 0))
        batches.append([key, wide, _payload(base, n)])
        base += n
    assert _run_ooc(b2, batches, [(0, 1, 0)], 16 << 10) > 1


def test_out_of_core_sort_multi_key(b2):
    rng = np.random.default_rng(11)
    batches, base = [], 0
    for b in range(7):
        n = int(rng.integers(0, 900))
        batches.append([O.OCol(rng.integers(0, 4, n).astype(np.int16), rng.random(n) >= 0.2, (O.INT16, 0, 0)),
                        O.OCol(rng.integers(-3, 3, n).astype(np.float32), np.ones(n, bool), (O.FLOAT32, 0, 0)),
                        O.OCol(_strings(rng, n, 5 if b % 2 else 60), np.ones(n, bool), (O.STRING, 0, 0)), _payload(base, n)])
        base += n
    _run_ooc(b2, batches, [(0, 0, 1), (1, 1, 0), (2, 1, 1)], 16 << 10)


def test_out_of_core_sort_no_empty_and_one_batch(b2):
    from spark_rapids_b200 import execs as E
    node = E.GpuSortExec([(0, 1, 1)], E.GpuBatchSource([]), target_bytes=1 << 20)
    assert list(node) == [] and node.metrics["numOutputRows"] == 0 and node.metrics["numOutputBatches"] == 0
    empty = [[O.OCol(np.zeros(0, np.int64), np.ones(0, bool), (O.INT64, 0, 0)), _payload(0, 0)] for _ in range(3)]
    assert _run_ooc(b2, empty, [(0, 1, 1)], 1 << 20) == 0
    one = [[O.OCol(np.array([5, 3, 9, 3], np.int64), np.ones(4, bool), (O.INT64, 0, 0)), _payload(0, 4)]]
    assert _run_ooc(b2, empty[:1] + one + empty[:1], [(0, 1, 1)], 1 << 20) == 1


# ---- 3. beyond device memory --------------------------------------------------------------------------------------------------
def _host_batches(keys, pays, rows):
    return [[(O.INT64, 0, keys[s:s + rows], None), (O.INT64, 0, pays[s:s + rows], None)] for s in range(0, len(keys), rows)]


def test_out_of_core_sort_beyond_the_allocation_limit(b2, limits):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(21)
    rows, nb = 1 << 17, 48                 # 48 batches of 2 MiB: 96 MiB of input
    keys = rng.integers(-2**40, 2**40, rows * nb).astype(np.int64)
    pays = np.arange(rows * nb, dtype=np.int64)
    b2.sync()
    base = b2.device_bytes_in_use()
    spilled0 = b2.memory_stats()["spilled_bytes"]
    b2.set_alloc_limit(base + (32 << 20))
    node = E.GpuSortExec([(0, 1, 1)], E.GpuHostBatchSource(_host_batches(keys, pays, rows)), target_bytes=4 << 20)
    got_k, got_p = [], []
    for t in node:
        assert _table_bytes(t) <= 4 << 20
        got_k.append(t.column(0).to_numpy()[0])
        got_p.append(t.column(1).to_numpy()[0])
        del t
    perm = np.argsort(keys, kind="stable")
    assert np.array_equal(np.concatenate(got_k), keys[perm]) and np.array_equal(np.concatenate(got_p), pays[perm])
    assert b2.memory_stats()["spilled_bytes"] > spilled0
    assert node.metrics["numOutputRows"] == rows * nb and node.metrics["numOutputBatches"] == len(got_k) > 1
    del node
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base
    single = E.GpuSortExec([(0, 1, 1)], E.GpuHostBatchSource(_host_batches(keys, pays, rows)))
    with pytest.raises(b2.B2Error) as ei:
        single.collect()
    assert ei.value.code == 3   # B2_ERR_OOM
    del single, ei
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base


# ---- 4. past 2^31 rows --------------------------------------------------------------------------------------------------------
def test_out_of_core_sort_past_2_31_rows(b2):
    """2^31 + 2^20 rows of (INT32 key in [0, 1000), INT32 payload = input position) in batches of 2^27 rows, checked one output
    batch at a time.  About 110 s on one H100 80GB HBM3 at a 700 W power limit, most of it generating and checking on the host."""
    from spark_rapids_b200 import execs as E
    n, rows = (1 << 31) + (1 << 20), 1 << 27
    rng = np.random.default_rng(31)
    keys = rng.integers(0, 1000, n, dtype=np.int32)
    pays = np.arange(n, dtype=np.uint32).view(np.int32)      # positions past 2^31 wrap; order is checked on the unsigned view
    batches = [[(O.INT32, 0, keys[s:s + rows], None), (O.INT32, 0, pays[s:s + rows], None)] for s in range(0, n, rows)]
    single = E.GpuSortExec([(0, 1, 1)], E.GpuHostBatchSource(batches))
    with pytest.raises(b2.B2Error) as ei:
        single.collect()
    assert ei.value.code == 4   # B2_ERR_SIZE_OVERFLOW
    del single, ei
    gc.collect()
    hist = sum(np.bincount(keys[s:s + rows], minlength=1000) for s in range(0, n, rows))
    want_sum = int(n) * (n - 1) // 2
    node = E.GpuSortExec([(0, 1, 1)], E.GpuHostBatchSource(batches), target_bytes=1 << 30)
    got_hist = np.zeros(1000, np.int64)
    got_sum, last_k, last_p, nout, nrows = 0, -1, -1, 0, 0
    for t in node:
        assert t.num_rows < 2**31
        k = t.column(0).to_numpy()[0].astype(np.int64)
        p = t.column(1).to_numpy()[0].view(np.uint32).astype(np.int64)
        del t
        assert k[0] > last_k or (k[0] == last_k and p[0] > last_p)
        assert np.all(np.diff(k) >= 0)
        same = np.diff(k) == 0
        assert np.all(np.diff(p)[same] > 0)
        got_hist += np.bincount(k, minlength=1000)
        got_sum += int(p.sum())
        last_k, last_p = int(k[-1]), int(p[-1])
        nout += 1
        nrows += len(k)
    assert nrows == n and nout > 1
    assert np.array_equal(got_hist, hist) and got_sum == want_sum
    assert node.metrics["numOutputRows"] == n and node.metrics["numOutputBatches"] == nout
