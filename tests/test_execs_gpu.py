"""Operator-layer (GpuExec mirror, csrc/exec.cu) parity: TPC-H q6 / q1 / q3 shaped plans built from
the reference's exec nodes, multi-batch, vs the oracle.  These read like the reference's
SparkQueryCompareTestSuite tests: same plan, CPU result == GPU result."""
import io

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from oracle import tpch
from tests import datagen as G

pytestmark = pytest.mark.gpu
DEC = (O.DECIMAL64, 12, 2)


def batches(b2, ocols, nb):
    n = len(ocols[0])
    cuts = [n * i // nb for i in range(nb + 1)]
    return [G.to_b2_table(b2, [O.OCol(c.values[a:b], c.valid[a:b], c.typ) for c in ocols]) for a, b in zip(cuts[:-1], cuts[1:])]


def test_q6_plan_from_parquet_multi_file(b2):
    from spark_rapids_b200 import execs as E
    import bench
    files = [tpch.lineitem_q6_parquet(40000, 100 + i, row_group_rows=15000) for i in range(3)]
    scan = E.GpuParquetScanExec(files, ["l_shipdate", "l_discount", "l_quantity", "l_extendedprice"])
    prog, spec = bench.build_q6(b2)
    partial = E.GpuHashAggregateExec(scan, [], spec, pre_project=[prog.exprs[1]], condition=prog.exprs[0])
    final = E.GpuHashAggregateExec(E.GpuShuffleExchangeExec(partial, []), [], spec, mode="final")
    got = final.collect().to_rows()
    exp = sum(tpch.q6_numpy_chunks(tpch.lineitem_q6_chunks(40000, 100 + i, 15000)) or 0 for i in range(3))
    assert got == [(exp,)]
    assert scan.metrics["numOutputRows"] == 120000 and scan.metrics["numOutputBatches"] == 3


def test_q1_plan_partial_exchange_final_sort(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(11)
    n = 40000
    rf = O.OCol(np.array([b"A", b"N", b"R"], dtype=object)[rng.integers(0, 3, n)], np.ones(n, bool), (O.STRING, 0, 0))
    ls = O.OCol(np.array([b"F", b"O"], dtype=object)[rng.integers(0, 2, n)], np.ones(n, bool), (O.STRING, 0, 0))
    qty = G.gen_column(rng, DEC, n, 0.0, distinct=50)
    price = G.gen_column(rng, DEC, n, 0.0, small=True)
    disc = G.gen_column(rng, DEC, n, 0.0, distinct=11)
    tax = G.gen_column(rng, DEC, n, 0.0, distinct=9)
    ship = O.OCol(rng.integers(8036, 10561, n).astype(np.int32), np.ones(n, bool), (O.DATE32, 0, 0))
    ocols = [rf, ls, qty, price, disc, tax, ship]
    c = [G.b2_expr_col(b2, i, oc) for i, oc in enumerate(ocols)]
    one = b2.lit(1, b2.DECIMAL32, 1, 0)
    pred = c[6] <= b2.lit(10471, b2.DATE32)
    disc_price = c[3] * (one - c[4])
    charge = disc_price * (one + c[5])
    pre = [c[0], c[1], c[2], c[3], disc_price, charge, c[4]]
    specs = [(O.AGG_SUM, 2, O.DECIMAL128, 2, 22), (O.AGG_SUM, 3, O.DECIMAL128, 2, 22), (O.AGG_SUM, 4, O.DECIMAL128, 4, 36),
             (O.AGG_SUM, 5, O.DECIMAL128, 6, 38), (O.AGG_COUNT, 2), (O.AGG_SUM, 6, O.DECIMAL128, 2, 22), (O.AGG_COUNT_ALL, 0)]
    src = E.GpuBatchSource(batches(b2, ocols, 4))
    partial = E.GpuHashAggregateExec(src, [0, 1], specs, pre_project=pre, condition=pred)
    final = E.GpuHashAggregateExec(E.GpuShuffleExchangeExec(partial, [0, 1]), [0, 1], specs, mode="final")
    out = E.GpuSortExec([(0, 1, 1), (1, 1, 1)], final).collect()
    keep = O.eval_expr(pred.sexpr, ocols)
    proj = O.filter_cols([O.eval_expr(e.sexpr, ocols) for e in pre], keep)
    exp_cols = O.groupby_cols(proj, [0, 1], specs)
    order = R.sort_order(exp_cols, [(0, 1, 1), (1, 1, 1)])
    assert out.to_rows() == O.rows_of(R.take(exp_cols, order))
    assert out.num_rows == 6


def test_q3_plan_joins_groupby_topn(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(3)
    nc, no, nl = 1500, 15000, 60000
    i64, i32, i8, date = (O.INT64, 0, 0), (O.INT32, 0, 0), (O.INT8, 0, 0), (O.DATE32, 0, 0)
    cust = [O.OCol(np.arange(nc, dtype=np.int64), np.ones(nc, bool), i64), O.OCol(rng.integers(0, 5, nc).astype(np.int8), np.ones(nc, bool), i8)]
    orders = [O.OCol(np.arange(no, dtype=np.int64) * 4, np.ones(no, bool), i64), O.OCol(rng.integers(0, nc, no).astype(np.int64), np.ones(no, bool), i64),
              O.OCol(rng.integers(8036, 10561, no).astype(np.int32), np.ones(no, bool), date), O.OCol(np.zeros(no, np.int32), np.ones(no, bool), i32)]
    line = [O.OCol(rng.integers(0, no, nl).astype(np.int64) * 4, np.ones(nl, bool), i64), G.gen_column(rng, DEC, nl, 0.0, small=True),
            G.gen_column(rng, DEC, nl, 0.0, distinct=11), O.OCol(rng.integers(8036, 10561, nl).astype(np.int32), np.ones(nl, bool), date)]
    D = 9204  # 1995-03-15
    # ---- plan (TPC-H q3; c_mktsegment is a dictionary code here: string predicates are a "next" row)
    cc = [G.b2_expr_col(b2, i, c) for i, c in enumerate(cust)]
    oc = [G.b2_expr_col(b2, i, c) for i, c in enumerate(orders)]
    lc = [G.b2_expr_col(b2, i, c) for i, c in enumerate(line)]
    cust_f = E.GpuFilterExec(cc[1] == b2.lit(1, b2.INT8), E.GpuBatchSource(batches(b2, cust, 1)))
    ord_f = E.GpuFilterExec(oc[2] < b2.lit(D, b2.DATE32), E.GpuBatchSource(batches(b2, orders, 2)))
    j1 = E.GpuShuffledHashJoinExec([1], [0], b2.JOIN_INNER, ord_f, cust_f)             # orders(4) ++ customer(2)
    line_f = E.GpuFilterExec(lc[3] > b2.lit(D, b2.DATE32), E.GpuBatchSource(batches(b2, line, 3)))
    j2 = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, line_f, E.GpuCoalesceBatches(j1, 1 << 30))   # line(4) ++ j1(6)
    one = b2.lit(1, b2.DECIMAL32, 1, 0)
    jl_price, jl_disc = b2.col(1, b2.DECIMAL64, 12, 2, nullable=False), b2.col(2, b2.DECIMAL64, 12, 2, nullable=False)
    pre = [b2.col(0, b2.INT64, nullable=False), b2.col(6, b2.DATE32, nullable=False), b2.col(7, b2.INT32, nullable=False), jl_price * (one - jl_disc)]
    specs = [(O.AGG_SUM, 3, O.DECIMAL128, 4, 36)]
    agg = E.GpuHashAggregateExec(j2, [0, 1, 2], specs, pre_project=pre, mode="complete")
    top = E.GpuTopN(10, [(3, 0, 0), (1, 1, 1)], agg)
    got = top.collect().to_rows()
    # ---- oracle
    ck = set(int(k) for k, s in zip(cust[0].values, cust[1].values) if s == 1)
    omap = {int(k): (int(d), int(p)) for k, c, d, p in zip(orders[0].values, orders[1].values, orders[2].values, orders[3].values) if d < D and int(c) in ck}
    rev = {}
    for k, p, dsc, sd in zip(line[0].values, line[1].values, line[2].values, line[3].values):
        if sd > D and int(k) in omap:
            key = (int(k),) + omap[int(k)]
            rev[key] = rev.get(key, 0) + int(p) * (100 - int(dsc))
    rows = sorted(((k[0], k[1], k[2], v) for k, v in rev.items()), key=lambda r: (-r[3], r[1]))[:10]
    assert [(r[3], r[1]) for r in got] == [(r[3], r[1]) for r in rows]     # order by revenue desc, o_orderdate
    assert sorted(got) == sorted(rows)
    assert j2.metrics["numOutputBatches"] == 3


def test_each_batch_sort_and_coalesce(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(5)
    c = G.gen_column(rng, (O.INT64, 0, 0), 10000, null_frac=0.1)
    src = E.GpuBatchSource(batches(b2, [c], 5))
    out = list(E.GpuSortExec([(0, 1, 1)], src, global_sort=False))
    assert len(out) == 5
    for t in out:
        vals = [v for v in t.column(0).to_pylist() if v is not None]
        assert vals == sorted(vals)
    co = list(E.GpuCoalesceBatches(E.GpuBatchSource(batches(b2, [c], 10)), 2500))
    assert [t.num_rows for t in co] == [2000, 2000, 2000, 2000, 2000]
    co2 = list(E.GpuCoalesceBatches(E.GpuBatchSource(batches(b2, [c], 10)), 10**9))
    assert [t.num_rows for t in co2] == [10000]


def test_full_outer_join_exec_multi_batch(b2):
    """GpuShuffledHashJoinExec FullOuter over a stream side that arrives in several batches: every stream row and
    every build row exactly once, the missing side NULL"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(8)
    i64 = (O.INT64, 0, 0)
    ns, nb = 9000, 2500
    stream = [O.OCol(rng.integers(0, 4000, ns).astype(np.int64), rng.random(ns) > 0.05, i64), O.OCol(np.arange(ns, dtype=np.int64), np.ones(ns, bool), i64)]
    build = [O.OCol(rng.permutation(6000)[:nb].astype(np.int64), rng.random(nb) > 0.05, i64), O.OCol(np.arange(nb, dtype=np.int64) + 10**6, np.ones(nb, bool), i64)]
    j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_FULL_OUTER, E.GpuBatchSource(batches(b2, stream, 4)), E.GpuBatchSource(batches(b2, build, 2)))
    got = sorted(j.collect().to_rows(), key=lambda r: tuple((x is None, x) for x in r))
    bmap = {int(k): int(v) for k, v, ok in zip(build[0].values, build[1].values, build[0].valid) if ok}
    exp, hit = [], set()
    for k, sid, ok in zip(stream[0].values, stream[1].values, stream[0].valid):
        if ok and int(k) in bmap:
            exp.append((int(k), int(sid), int(k), bmap[int(k)])); hit.add(int(k))
        else:
            exp.append((int(k) if ok else None, int(sid), None, None))
    for k, v, ok in zip(build[0].values, build[1].values, build[0].valid):
        if not ok or int(k) not in hit:
            exp.append((None, None, int(k) if ok else None, int(v)))
    exp = sorted(exp, key=lambda r: tuple((x is None, x) for x in r))
    assert got == exp


def _q3_small(b2, sf, host):
    """the SF100 bench plan (bench.build_q3_plan) on a small instance of the same generator vs the numpy restatement"""
    from spark_rapids_b200 import execs as E
    import bench
    chunks = bench.q3_host_chunks(sf, 0, 1)
    progs = bench.q3_programs(b2)
    if host:
        hb = bench.q3_host_batches(b2, chunks)
        src = {t: E.GpuHostBatchSource(hb[t]) for t in bench.Q3_SCHEMA}
    else:
        dev = bench.q3_device_batches(b2, chunks)
        src = {t: E.GpuBatchSource(dev[t]) for t in bench.Q3_SCHEMA}
    root, nodes = bench.build_q3_plan(b2, E, progs, src)
    got = bench.q3_rows_of(root.collect())
    exp = tpch.q3_expected(sf, 42, threads=4)
    assert [(r[1], r[2]) for r in got] == [(r[1], r[2]) for r in exp]
    assert sorted(got) == sorted(exp)
    assert nodes["filter_lineitem"].metrics["numOutputBatches"] == 16 and nodes["join_lineitem_orders"].metrics["numOutputBatches"] == 16
    return nodes


def test_q3_bench_plan_small_resident(b2):
    _q3_small(b2, 0.05, False)


def test_q3_bench_plan_small_host_batches(b2):
    """HostColumnarToGpu: the same plan fed from host column batches (pageable here; the bench pins them)"""
    _q3_small(b2, 0.02, True)


def test_join_exec_output_pruning(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(21)
    i64 = (O.INT64, 0, 0)
    ns, nb = 5000, 800
    stream = [O.OCol(rng.integers(0, 1000, ns).astype(np.int64), np.ones(ns, bool), i64), O.OCol(np.arange(ns, dtype=np.int64), np.ones(ns, bool), i64)]
    build = [O.OCol(np.arange(nb, dtype=np.int64), np.ones(nb, bool), i64), O.OCol(np.arange(nb, dtype=np.int64) * 7, np.ones(nb, bool), i64)]
    full = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource(batches(b2, stream, 3)), E.GpuBatchSource(batches(b2, build, 1))).collect()
    pruned = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource(batches(b2, stream, 3)), E.GpuBatchSource(batches(b2, build, 1)),
                                       stream_out=[1], build_out=[1]).collect()
    assert sorted((r[1], r[3]) for r in full.to_rows()) == sorted(pruned.to_rows())
    only_stream = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource(batches(b2, stream, 3)), E.GpuBatchSource(batches(b2, build, 1)),
                                            stream_out=[1], build_out=[]).collect()
    assert sorted(r[0] for r in only_stream.to_rows()) == sorted(r[1] for r in full.to_rows())


@pytest.mark.parametrize("keytype", ["int64", "int32"])
def test_filter_fused_into_probe(b2, keytype, monkeypatch):
    """GpuFilter below the stream side of an INNER FK -> PK join: a simple predicate evaluated inside the probe kernel
    (opt-in, B2_JOIN_PRED_FUSION: measured slower on q3), the selection-vector path (default) and the unfused plan give the
    same rows, and all equal numpy"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(77)
    ns, nb = 300_000, 400_000                                  # >= 2^18 build rows: the Bloom filter is on
    kt = np.int64 if keytype == "int64" else np.int32
    skey = rng.integers(0, 1_000_000, ns).astype(kt)           # ~40 % of the stream keys exist on the build side
    sdate = rng.integers(8000, 11000, ns).astype(np.int32)
    sval = rng.integers(0, 1 << 40, ns).astype(np.int64)
    bkey = rng.permutation(1_000_000)[:nb].astype(kt)
    bval = (bkey.astype(np.int64) * 3 + 1)

    def plan():
        st = b2.Table.from_columns([b2.Column.from_numpy(skey), b2.Column.from_numpy(sdate, dtype=b2.DATE32), b2.Column.from_numpy(sval)])
        bt = b2.Table.from_columns([b2.Column.from_numpy(bkey), b2.Column.from_numpy(bval)])
        half = ns // 2
        srcs = E.GpuBatchSource([b2.slice_table(st, 0, half), b2.slice_table(st, half, ns)])
        pred = b2.Program([(b2.col(1, b2.DATE32, nullable=False) > b2.lit(9204, b2.DATE32)) & (b2.col(2, b2.INT64, nullable=False) >= b2.lit(1 << 20, b2.INT64))])
        flt = E.GpuFilterExec(pred, srcs)
        return E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, flt, E.GpuBatchSource([bt]), stream_out=[0, 2], build_out=[1]), flt

    keep = (sdate > 9204) & (sval >= (1 << 20))
    lut = np.full(1_000_000, -1, dtype=np.int64)
    lut[bkey.astype(np.int64)] = bval
    hit = keep & (lut[skey.astype(np.int64)] >= 0)
    want = sorted(zip(skey[hit].tolist(), sval[hit].tolist(), lut[skey[hit].astype(np.int64)].tolist()))
    for env in ({"B2_JOIN_PRED_FUSION": "1"}, {}, {"B2_NO_FILTER_FUSION": "1"}):
        for k in ("B2_JOIN_PRED_FUSION", "B2_NO_FILTER_FUSION"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        j, flt = plan()
        out = j.collect()
        assert sorted(out.to_rows()) == want, env
        assert flt.metrics["numOutputRows"] == int(keep.sum()), env


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_mixed_join_condition(b2, kind):
    """Table.mixed*JoinGatherMaps (GpuHashJoin.scala:335-600): equi keys + a non-equi condition over both sides
    (TPC-H q21 shape: l2.l_orderkey = l1.l_orderkey AND l2.l_suppkey <> l1.l_suppkey), vs a nested-loop restatement"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(50 + kind)
    i64 = (O.INT64, 0, 0)
    ns, nb = 4000, 1500
    stream = [O.OCol(rng.integers(0, 600, ns).astype(np.int64), rng.random(ns) > 0.03, i64), O.OCol(rng.integers(0, 8, ns).astype(np.int64), np.ones(ns, bool), i64),
              O.OCol(np.arange(ns, dtype=np.int64), np.ones(ns, bool), i64)]
    build = [O.OCol(rng.integers(0, 600, nb).astype(np.int64), rng.random(nb) > 0.03, i64), O.OCol(rng.integers(0, 8, nb).astype(np.int64), rng.random(nb) > 0.1, i64)]
    cond = b2.col(1, b2.INT64) != b2.col(4, b2.INT64)          # stream.supp <> build.supp (pair columns: 3 stream ++ 2 build)
    j = E.GpuShuffledHashJoinExec([0], [0], kind, E.GpuBatchSource(batches(b2, stream, 3)), E.GpuBatchSource(batches(b2, build, 2)), condition=cond)
    out = j.collect()
    got = out.to_rows() if out is not None else []
    exp = []
    bk = {}
    for k, s, ok, sok in zip(build[0].values, build[1].values, build[0].valid, build[1].valid):
        if ok:
            bk.setdefault(int(k), []).append((int(k), int(s) if sok else None))
    for k, s, i, ok in zip(stream[0].values, stream[1].values, stream[2].values, stream[0].valid):
        srow = (int(k) if ok else None, int(s), int(i))
        hits = [b for b in bk.get(int(k), [])] if ok else []
        passing = [b for b in hits if b[1] is not None and b[1] != int(s)]     # NULL <> x is NULL -> not a match
        if kind == 0:
            exp += [srow + b for b in passing]
        elif kind == 1:
            exp += [srow + b for b in passing] if passing else [srow + (None, None)]
        elif kind == 2 and passing:
            exp.append(srow)
        elif kind == 3 and not passing:
            exp.append(srow)
    key = lambda r: tuple((x is None, x) for x in r)
    assert sorted(got, key=key) == sorted(exp, key=key)


def test_expand_exec_two_count_distincts(b2):
    """GpuExpandExec: the plan shape of `select count(distinct a), count(distinct b)`: expand to (a, NULL, 1) / (NULL, b, 2),
    group by (a, b, gid), then count per gid"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(31)
    i64, i32 = (O.INT64, 0, 0), (O.INT32, 0, 0)
    n = 5000
    a, b = G.gen_column(rng, i64, n, distinct=37, null_frac=0.1), G.gen_column(rng, i64, n, distinct=91, null_frac=0.05)
    ca, cb = G.b2_expr_col(b2, 0, a), G.b2_expr_col(b2, 1, b)
    null64 = b2.lit(None, b2.INT64)
    ex = E.GpuExpandExec([[ca, null64, b2.lit(1, b2.INT32)], [null64, cb, b2.lit(2, b2.INT32)]], E.GpuBatchSource(batches(b2, [a, b], 3)))
    rows = [r for t in ex for r in t.to_rows()]
    assert len(rows) == 2 * n
    exp = [(x, None, 1) for x in a.to_pylist()] + [(None, y, 2) for y in b.to_pylist()]
    key = lambda r: tuple((x is None, x) for x in r)
    assert sorted(rows, key=key) == sorted(exp, key=key)
    da = len({x for x in a.to_pylist() if x is not None}); db = len({y for y in b.to_pylist() if y is not None})
    distinct = {r for r in rows}
    assert sum(1 for r in distinct if r[2] == 1 and r[0] is not None) == da and sum(1 for r in distinct if r[2] == 2 and r[1] is not None) == db


def _dec_batches(b2, rows_per_batch, nullable):
    """batches of (INT64 key, DECIMAL128(38,0) value) rows; a value of None is NULL"""
    out = []
    for rows in rows_per_batch:
        k = np.array([r[0] for r in rows], dtype=np.int64)
        v = np.array([0 if r[1] is None else r[1] for r in rows], dtype=object)
        ok = np.array([r[1] is not None for r in rows])
        out.append(b2.Table.from_columns([b2.Column.from_numpy(k), b2.Column.from_numpy(v, dtype=b2.DECIMAL128, valid=ok if nullable else None)]))
    return out


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("keyed", [True, False])
@pytest.mark.parametrize("plan", ["complete", "partial_exchange_final"])
def test_decimal_sum_overflow_in_one_batch_stays_null(b2, plan, keyed, nullable):
    """SUM(d), d DECIMAL(38,0), result precision 38, over two batches.  Key 1: batch 1 holds 6e37 + 6e37 (its partial
    overflows, NULL), batch 2 holds 1: Spark's result is NULL (buffer (sum, isEmpty): sum NULL and isEmpty false), and so
    is the exact total.  A merge that skipped the NULL partial would return 1.  Key 2 sums normally; key 3 (nullable
    input) has only a NULL in batch 1, an empty partial that the merge must skip.
    Not pinned: a batch that overflows while the exact total fits (6e37 + 6e37 - 6e37).  This gives NULL, but Spark
    makes no promise there (its partial sums may or may not overflow depending on how the input is split)."""
    from spark_rapids_b200 import execs as E
    big = 6 * 10**37
    if keyed:
        b1 = [(1, big), (1, big), (2, 5)] + ([(3, None)] if nullable else [])
        b2_ = [(1, 1), (2, 7), (3, 4)]
        want = [(1, None), (2, 12), (3, 4)]
    else:
        b1 = [(0, big), (0, big)] + ([(0, None)] if nullable else [])
        b2_ = [(0, 1)]
        want = [(None,)]
    keys = [0] if keyed else []
    spec = [(b2.AGG_SUM, len(keys), b2.DECIMAL128, 0, 38)]
    pre = ([b2.col(0, b2.INT64, nullable=False)] if keyed else []) + [b2.col(1, b2.DECIMAL128, 38, 0, nullable=nullable)]
    src = E.GpuBatchSource(_dec_batches(b2, [b1, b2_], nullable))
    if plan == "complete":
        root = E.GpuHashAggregateExec(src, keys, spec, pre_project=pre, mode="complete")
    else:
        partial = E.GpuHashAggregateExec(src, keys, spec, pre_project=pre)
        root = E.GpuHashAggregateExec(E.GpuShuffleExchangeExec(partial, keys), keys, spec, mode="final")
    out = root.collect()
    assert out.num_columns == len(keys) + 1
    assert sorted(out.to_rows(), key=lambda r: r[0] if keyed else 0) == want


@pytest.mark.parametrize("plan", ["complete", "partial_exchange_final"])
def test_nullable_decimal_sum_empty_partials_are_skipped(b2, plan):
    """keyless SUM over a nullable column whose first batch is all NULL: that partial is empty, not an overflow"""
    from spark_rapids_b200 import execs as E
    spec = [(b2.AGG_SUM, 0, b2.DECIMAL128, 0, 38)]
    pre = [b2.col(1, b2.DECIMAL128, 38, 0, nullable=True)]
    src = E.GpuBatchSource(_dec_batches(b2, [[(0, None), (0, None)], [(0, 3)], [(0, None)]], True))
    if plan == "complete":
        root = E.GpuHashAggregateExec(src, [], spec, pre_project=pre, mode="complete")
    else:
        root = E.GpuHashAggregateExec(E.GpuShuffleExchangeExec(E.GpuHashAggregateExec(src, [], spec, pre_project=pre), []), [], spec, mode="final")
    assert root.collect().to_rows() == [(3,)]
