"""The emitting FK -> PK probe (join_filter_probe_kernel writing the output rows, GpuShuffledHashJoinExec.try_emit): the same
rows, as a multiset, as numpy and as the maps path (B2_JOIN_NO_EMIT, in a child process), the same numOutputRows on the filter
and the join, and which path each batch took (HashJoinExec.emit_stats)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 9204


def make_case(seed, key64, nbuild, batch_rows, nullable_build=False, pass_frac=None):
    """stream batches [key, date, v8, v4] and the build table [key, b4, b8, b4b, b8b] as numpy arrays"""
    rng = np.random.default_rng(seed)
    kt = np.int64 if key64 else np.int32
    dom = 4 * nbuild
    bkey = rng.permutation(dom)[:nbuild].astype(kt) + (kt(1) << 40 if key64 else 0)
    build = [bkey, rng.integers(-2**31, 2**31, nbuild).astype(np.int32), rng.integers(-2**63, 2**63, nbuild, dtype=np.int64),
             rng.integers(-2**31, 2**31, nbuild).astype(np.int32), rng.integers(-2**63, 2**63, nbuild, dtype=np.int64)]
    batches = []
    for i, n in enumerate(batch_rows):
        key = rng.choice(bkey, n) if i % 2 else rng.integers(0, dom, n).astype(kt) + (kt(1) << 40 if key64 else 0)
        frac = 0.5 if pass_frac is None else pass_frac[i]
        date = np.where(rng.random(n) < frac, D + 1 + rng.integers(0, 500, n), D - rng.integers(0, 500, n)).astype(np.int32)
        batches.append([key.astype(kt), date, rng.integers(-2**63, 2**63, n, dtype=np.int64), rng.integers(-2**31, 2**31, n).astype(np.int32)])
    return batches, build, nullable_build


def expected(batches, build, stream_out, build_out):
    lut = {int(k): i for i, k in enumerate(build[0])}
    rows = []
    for b in batches:
        keep = b[1] > D
        for r in np.flatnonzero(keep):
            br = lut.get(int(b[0][r]))
            if br is not None:
                rows.append(tuple(int(b[c][r]) for c in stream_out) + tuple(int(build[c][br]) for c in build_out))
    return sorted(rows)


def run(b2, case, stream_out, build_out):
    """-> (sorted rows, emit_stats, filter numOutputRows, join numOutputRows)"""
    from spark_rapids_b200 import execs as E
    batches, build, nullable_build = case
    st = [b2.Table.from_columns([b2.Column.from_numpy(c, dtype=b2.DATE32 if j == 1 else None) for j, c in enumerate(b)]) for b in batches]
    valid = np.ones(len(build[0]), bool)
    valid[::7] = False
    bt = b2.Table.from_columns([b2.Column.from_numpy(c, valid=valid if (nullable_build and j == 1) else None) for j, c in enumerate(build)])
    flt = E.GpuFilterExec(b2.Program([b2.col(1, b2.DATE32, nullable=False) > b2.lit(D, b2.DATE32)]), E.GpuBatchSource(st))
    j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, flt, E.GpuBatchSource([bt]), stream_out=stream_out, build_out=build_out)
    rows = []
    for t in j:
        rows += [tuple(x) for x in t.to_rows()]
    return sorted(rows), j.emit_stats, flt.metrics["numOutputRows"], j.metrics["numOutputRows"]


CASES = {
    # name: (make_case kwargs, stream_out, build_out)
    "i64_key_first_b8": (dict(seed=1, key64=True, nbuild=300_000, batch_rows=[70_000, 90_000, 80_000]), [0, 2, 3], [3, 1]),
    "i32_key_last_b4": (dict(seed=2, key64=False, nbuild=200_000, batch_rows=[70_000, 90_000, 80_000]), [3, 0], [1]),
    "i64_no_key_b16": (dict(seed=3, key64=True, nbuild=100_000, batch_rows=[66_000, 100_000]), [2, 3], [2, 3, 1]),
    "i32_key_mid_b16_one": (dict(seed=4, key64=False, nbuild=400_000, batch_rows=[80_000, 80_000]), [2, 0, 3], [4, 2]),
    "i64_build_empty": (dict(seed=5, key64=True, nbuild=50_000, batch_rows=[70_000, 70_000, 70_000]), [0, 2, 3], []),
    "i32_stream_empty": (dict(seed=6, key64=False, nbuild=300_000, batch_rows=[70_000, 70_000]), [], [2, 1]),
}


def child_rows(name):
    """the rows of CASES[name] through the maps path, in a child process with B2_JOIN_NO_EMIT set"""
    env = dict(os.environ, B2_JOIN_NO_EMIT="1")
    code = "import json, sys; sys.path.insert(0, %r); from tests import test_join_emit_gpu as t; t._child(%r)" % (ROOT, name)
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    return [tuple(x) for x in out["rows"]], out["stats"], out["npass"], out["nout"]


def _child(name):
    import spark_rapids_b200 as b2
    b2.init(0)
    kw, so, bo = CASES[name]
    rows, stats, npass, nout = run(b2, make_case(**kw), so, bo)
    print(json.dumps({"rows": rows, "stats": stats, "npass": npass, "nout": nout}))


@pytest.mark.parametrize("name", sorted(CASES))
def test_emit_matches_maps_and_numpy(b2, name):
    kw, so, bo = CASES[name]
    case = make_case(**kw)
    s0 = b2.memory_stats()["in_use"]
    rows, stats, npass, nout = run(b2, case, so, bo)
    assert b2.memory_stats()["in_use"] == s0
    nb = len(kw["batch_rows"])
    assert stats == {"emitted": nb - 1, "maps": 1, "overflows": 0}, stats
    want = expected(case[0], case[1], so, bo)
    assert rows == want and nout == len(want)
    assert npass == sum(int((b[1] > D).sum()) for b in case[0])
    mrows, mstats, mnpass, mnout = child_rows(name)
    assert mstats == {"emitted": 0, "maps": nb, "overflows": 0}, mstats
    assert mrows == rows and (mnpass, mnout) == (npass, nout)


@pytest.mark.parametrize("what", ["build_20_bytes", "build_nullable", "build_1_byte_wide", "stream_4_columns", "small_batches"])
def test_fallback_to_maps(b2, what):
    kw = dict(seed=7, key64=True, nbuild=100_000, batch_rows=[70_000, 70_000])
    so, bo = [0, 2], [1]
    if what == "build_20_bytes":
        bo = [2, 4, 1]
    elif what == "build_nullable":
        kw["nullable_build"] = True
    elif what == "stream_4_columns":
        so = [3, 2, 0, 3]
    elif what == "small_batches":
        kw["batch_rows"] = [40_000, 50_000, 60_000]
    case = make_case(**kw)
    if what == "build_1_byte_wide":   # an INT8 build column: 4- and 8-byte columns only
        case[1].append(case[1][1].astype(np.int8))
        bo = [5]
    rows, stats, npass, nout = run(b2, case, so, bo)
    assert stats == {"emitted": 0, "maps": len(case[0]), "overflows": 0}, stats
    want = expected(case[0], [c.astype(np.int64) if c.dtype == np.int8 else c for c in case[1]], so, bo)
    if what == "build_nullable":   # b4 (column 1) is NULL on every 7th build row
        lut = {int(k): i for i, k in enumerate(case[1][0])}
        want = sorted(r[:-1] + ((None,) if lut[r[0]] % 7 == 0 else (r[-1],)) for r in want)
    assert rows == want and nout == len(want)


def test_overflow_reruns_through_maps(b2):
    """the first batch passes 1 % of its rows, the second all of them: the second overflows its estimate and is joined again"""
    kw = dict(seed=8, key64=True, nbuild=300_000, batch_rows=[100_000, 400_000], pass_frac=[0.01, 1.0])
    case = make_case(**kw)
    case[0][1][0] = np.random.default_rng(9).choice(case[1][0], 400_000)   # every row of batch 2 matches
    so, bo = [0, 2], [1, 3]
    s0 = b2.memory_stats()["in_use"]
    rows, stats, npass, nout = run(b2, case, so, bo)
    assert b2.memory_stats()["in_use"] == s0
    assert stats == {"emitted": 0, "maps": 2, "overflows": 1}, stats
    want = expected(case[0], case[1], so, bo)
    assert rows == want and nout == len(want) > 400_000 * 0.99
    assert npass == sum(int((b[1] > D).sum()) for b in case[0])


def test_q3_plan_emits_after_first_batch(b2):
    """the bench's q3 plan on a small instance: each join takes the maps for its first batch and emits the rest"""
    sys.path.insert(0, ROOT)
    import bench
    from oracle import tpch
    from spark_rapids_b200 import execs as E
    sf = 0.1
    chunks = bench.q3_host_chunks(sf, 0, 1)
    for t, k in (("orders", 2), ("lineitem", 3)):   # k batches of at least 2^16 rows, the smallest the fused probe takes
        whole = {c: np.concatenate([ch[c] for ch in chunks[t]]) for c in chunks[t][0]}
        chunks[t] = [{c: v[i::k].copy() for c, v in whole.items()} for i in range(k)]
    dev = bench.q3_device_batches(b2, chunks)
    root, nodes = bench.build_q3_plan(b2, E, bench.q3_programs(b2), {t: E.GpuBatchSource(dev[t]) for t in bench.Q3_SCHEMA})
    got = bench.q3_rows_of(root.collect())
    exp = tpch.q3_expected(sf, 42, threads=2)
    for name, t in (("join_orders_customer", "orders"), ("join_lineitem_orders", "lineitem")):
        nb = len(chunks[t])
        assert all(len(ch[Q3_KEY[t]]) >= 1 << 16 for ch in chunks[t]), t
        assert nodes[name].emit_stats == {"emitted": nb - 1, "maps": 1, "overflows": 0}, (name, nodes[name].emit_stats)
    assert sorted(got) == sorted(exp)


Q3_KEY = {"orders": "o_custkey", "lineitem": "l_orderkey"}
