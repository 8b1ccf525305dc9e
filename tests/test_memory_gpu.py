"""(f4) memory-pressure contract and the threading contract of the boundary (SURVEY §8b): retryable OOM, spill store,
split-and-retry in the join / aggregate execs, GpuSemaphore, re-entrancy from several host threads."""
import gc
import threading

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from tests import datagen as G

pytestmark = pytest.mark.gpu
I64 = (O.INT64, 0, 0)


def _col(vals):
    return O.OCol(np.asarray(vals, dtype=np.int64), np.ones(len(vals), bool), I64)


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)
    b2.semaphore_init(0)


def test_oom_is_retryable_and_leaks_nothing(b2, limits):
    """RmmSpark.forceRetryOOM analogue: an allocation over the limit surfaces as B2_ERR_OOM (GpuRetryOOM); after the limit is
    lifted the same call succeeds and no device memory was leaked by the failed attempt"""
    n = 1 << 20
    t = G.to_b2_table(b2, [_col(np.arange(n) % 1000), _col(np.arange(n))])
    b2.sync()
    base = b2.device_bytes_in_use()
    b2.set_alloc_limit(base + (1 << 20))          # 1 MiB of headroom: the sort needs ~24 MiB
    with pytest.raises(b2.B2Error) as ei:
        b2.order_by(t, [(0, 1, 1)])
    assert ei.value.code == 3                     # B2_ERR_OOM
    b2.sync()
    assert b2.device_bytes_in_use() == base
    b2.set_alloc_limit(0)
    out = b2.order_by(t, [(0, 1, 1)])
    assert out.num_rows == n
    del out
    b2.sync()
    assert b2.device_bytes_in_use() == base


def test_spill_store_moves_batches_to_host_and_back(b2, limits):
    rng = np.random.default_rng(4)
    cols = [G.gen_column(rng, I64, 200000), G.gen_column(rng, (O.STRING, 0, 0), 200000), G.gen_column(rng, (O.DECIMAL128, 30, 2), 200000)]
    t = G.to_b2_table(b2, cols)
    sp = b2.Spillable(t)
    held = sp.get()
    assert b2.spill() == 0 and not sp.spilled      # a batch somebody holds is not spillable
    del held, t
    b2.sync()
    before = b2.device_bytes_in_use()
    freed = b2.spill()
    assert freed > 0 and sp.spilled and b2.device_bytes_in_use() <= before - freed + 4096
    back = sp.get()                               # unspill on access
    assert not sp.spilled
    for i, c in enumerate(cols):
        G.assert_col_equal(back.column(i), c)
    st = b2.memory_stats()
    assert st["spilled_bytes"] >= freed and st["unspilled_bytes"] >= freed
    sp.close()


def test_allocation_failure_spills_before_failing(b2, limits):
    """DeviceMemoryEventHandler: an allocation that does not fit first evicts spillable batches"""
    n = 1 << 20
    big = b2.Spillable(G.to_b2_table(b2, [_col(np.arange(n)), _col(np.arange(n))]))     # 16 MiB, nobody holds it
    b2.sync()
    b2.set_alloc_limit(b2.device_bytes_in_use() + (4 << 20))
    t = G.to_b2_table(b2, [_col(np.arange(n))])                                          # needs 8 MiB: only fits after the spill
    assert big.spilled and t.num_rows == n
    b2.set_alloc_limit(0)
    assert big.get().num_rows == n
    big.close()


def test_join_exec_splits_and_retries_under_memory_pressure(b2, limits):
    from spark_rapids_b200 import execs as E
    ns, nb = 1 << 19, 1 << 12
    rng = np.random.default_rng(6)
    stream = [_col(rng.integers(0, nb, ns)), _col(np.arange(ns))]
    build = [_col(np.arange(nb)), _col(np.arange(nb) * 3)]
    st, bt = G.to_b2_table(b2, stream), G.to_b2_table(b2, build)
    ref = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource([st]), E.GpuBatchSource([bt])).collect()
    exp = sorted(ref.to_rows())
    del ref
    b2.sync()
    s0 = b2.memory_stats()
    # the whole stream batch needs 2 x 2 MiB of maps + 4 x 4 MiB of gathered columns = 20 MiB at its peak; 14 MiB force a split
    # (each half peaks at 10 MiB + its 4 MiB slice; the consumer drops every output batch before asking for the next)
    b2.set_alloc_limit(b2.device_bytes_in_use() + (15 << 20))
    j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource([st]), E.GpuBatchSource([bt]))
    got, nout = [], 0
    while True:
        t = j.next()
        if t is None:
            break
        b2.set_alloc_limit(0)           # reading the batch back needs no device memory, but keep the limit out of the way
        got += t.to_rows(); nout += 1
        del t
        b2.sync()
        b2.set_alloc_limit(b2.device_bytes_in_use() + (15 << 20))
    b2.set_alloc_limit(0)
    s1 = b2.memory_stats()
    assert s1["splits"] > s0["splits"] and nout >= 2, (s0, s1, nout)
    assert sorted(got) == exp


def test_aggregate_splits_a_batch_under_memory_pressure(b2, limits):
    """COMPLETE-mode SUM and COUNT by an INT64 key over one batch of n = 2^22 rows (16 B per row), each key about four times.
    A first pass over more than 2^20 rows takes scan_aggregate's radix path: two row arrays of 20 B per row (hash, key, value),
    28 B per row of group slots (key, two accumulator words, validity word), about 1 B per row of tile counts, 24 B per group
    of output and the 2.25 MiB table of the cardinality probe.  Above what is in use with the batch, in B per row of the batch:
    the whole batch's first pass needs about 77; the split, both halves beside the batch, 16; each half's first pass, with the
    two halves (or one half and a partial) in place of the batch, about 36 + 5; the merge of the two partials (about 0.43 n
    rows), once the batch is gone, about 31.  A limit of 60 forces one split, and the halves' partials merge to the whole's
    result."""
    from spark_rapids_b200 import execs as E
    n = 1 << 22
    rng = np.random.default_rng(12)
    keys, vals = rng.integers(0, n // 4, n), rng.integers(-10**9, 10**9, n)
    src = E.GpuBatchSource([b2.Table.from_columns([b2.Column.from_numpy(keys), b2.Column.from_numpy(vals)])])
    pre = [b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.INT64, nullable=False)]
    specs = [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]
    node = E.GpuHashAggregateExec(src, [0], specs, pre_project=pre, mode="complete")
    del src
    gc.collect()
    b2.sync()
    s0 = b2.memory_stats()
    b2.set_alloc_limit(b2.device_bytes_in_use() + 60 * n)
    out = node.next()
    b2.set_alloc_limit(0)
    assert node.next() is None
    s1 = b2.memory_stats()
    assert s1["splits"] > s0["splits"], (s0, s1)
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    k, s, c = (out.column(i).to_numpy()[0] for i in range(3))
    o = np.argsort(k)
    assert np.array_equal(k[o], sk[starts])
    assert np.array_equal(s[o], np.add.reduceat(vals[order], starts))
    assert np.array_equal(c[o], np.diff(np.r_[starts, n]))


def test_semaphore_bounds_concurrent_tasks(b2, limits):
    b2.semaphore_init(2)
    inside, peak, lock = [0], [0], threading.Lock()

    def task():
        b2.semaphore_acquire()
        with lock:
            inside[0] += 1; peak[0] = max(peak[0], inside[0])
        t = G.to_b2_table(b2, [_col(np.arange(200000))])
        b2.filter_count(b2.Program([b2.col(0, b2.INT64, nullable=False) > b2.lit(5, b2.INT64)]), t)
        with lock:
            inside[0] -= 1
        b2.semaphore_release()
    th = [threading.Thread(target=task) for _ in range(8)]
    [x.start() for x in th]; [x.join() for x in th]
    st = b2.semaphore_stats()
    assert peak[0] <= 2 and st["holders"] == 0 and st["permits"] == 2


def test_boundary_is_reentrant_from_many_threads(b2):
    """SURVEY §8b threading: many task threads, each on its own stream, results equal to the serial ones"""
    def work(seed):
        rng = np.random.default_rng(seed)
        n = 150000
        k = G.gen_column(rng, I64, n, distinct=97)
        v = G.gen_column(rng, (O.DECIMAL64, 12, 2), n, small=True)
        t = G.to_b2_table(b2, [k, v])
        ck, cv = G.b2_expr_col(b2, 0, k), G.b2_expr_col(b2, 1, v)
        f = b2.filter(b2.Program([ck > b2.lit(10, b2.INT64)]), t)
        g = b2.groupby(f, [0], [(O.AGG_SUM, 1, O.DECIMAL128, 2, 22), (O.AGG_COUNT_ALL, 0)])
        s = b2.order_by(g, [(0, 1, 1)])
        ht = b2.JoinHashTable(b2.Table.from_columns([s.column(0)]))
        lm, rm = ht.probe(b2.Table.from_columns([t.column(0)]), 0)
        return s.to_rows(), len(lm)
    serial = [work(s) for s in range(4)]
    out = [None] * 4

    def run(i):
        out[i] = work(i)
    th = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    [x.start() for x in th]; [x.join() for x in th]
    assert out == serial
