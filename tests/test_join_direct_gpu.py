"""The direct join table (join.cu): a build side of one distinct integer key column whose span R = max - min + 1 is at most
2^28 and at most 64 x its non-NULL keys is stored as an exact bitmap over [min, min + R) with a rank per 256-bit block, and
the one-key probes find a key's build row through its rank instead of the hash table.  Every probe path is checked against
the exact numpy reference of test_join_paths_gpu.py; which layout was built shows in the kernel timings
(join_direct_rows_kernel for the direct layout, join_build_kernel for the hash table, also when a direct table builds it
on the first probe that has no direct variant)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import spark_cpu as O
from tests.test_build_outer_join_gpu import assert_right_outer, right_outer_maps
from tests.test_join_paths_gpu import assert_maps, join_maps, join_maps_all, ocol, to_table

pytestmark = pytest.mark.gpu

INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER, RIGHT_OUTER = range(6)
DIRECT_BUILD, HASH_BUILD = "join_direct_rows_kernel", "join_build_kernel"
ONE_KEY = "join_probe_distinct1_kernel"
TYPE_RANGE = {O.INT32: (-2**31, 2**31 - 1), O.DATE32: (-2**31, 2**31 - 1), O.DECIMAL32: (-2**31, 2**31 - 1), O.INT64: (-2**63, 2**63 - 1),
              O.TIMESTAMP_US: (-2**63, 2**63 - 1), O.DECIMAL64: (-2**63, 2**63 - 1)}


def profiled(b2, fn):
    b2.profile_enable(True)
    try:
        out = fn()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return out, names


def build(b2, cols, nulls_equal=False):
    """-> (hash table, "direct" | "hash")"""
    ht, names = profiled(b2, lambda: b2.JoinHashTable(to_table(b2, cols), nulls_equal))
    direct = DIRECT_BUILD in names
    assert direct != (HASH_BUILD in names), names
    return ht, "direct" if direct else "hash"


def probe(b2, ht, pt, kind, selection=None):
    (lm, rm), names = profiled(b2, lambda: ht.probe(pt, kind, selection=selection))
    return (lm.to_numpy()[0].astype(np.int64), None if rm is None else rm.to_numpy()[0].astype(np.int64)), names


def typed(values, typ):
    return ocol(np.asarray(values, np.int64 if TYPE_RANGE[typ][1] > 2**31 else np.int32), (typ, 0, 2 if typ in (O.DECIMAL32, O.DECIMAL64) else 0))


def edge_probe_keys(rng, bkeys, typ):
    """present keys, absent keys inside the span, min - 1, max + 1, the type's extremes, and every 64-bit word and 256-bit
    block boundary of the bitmap"""
    lo, hi = int(bkeys.min()), int(bkeys.max())
    tmin, tmax = TYPE_RANGE[typ]
    span = hi - lo + 1
    extra = [lo + b + d for b in range(0, span + 64, 64) for d in (-1, 0, 1, 63)]
    extra += [lo - 1, hi + 1, lo - 2**20, hi + 2**20, tmin, tmax, tmin + 1, tmax - 1, 0, -1]
    extra = np.array([x for x in extra if tmin <= x <= tmax], np.int64)
    k = np.concatenate([rng.choice(bkeys, 3 * len(bkeys)).astype(np.int64), rng.integers(lo, hi, 2 * len(bkeys), dtype=np.int64, endpoint=True), extra])
    return k[rng.permutation(len(k))]


# ---- 1. every probe path on a direct table --------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", [O.INT64, O.INT32, O.DATE32, O.DECIMAL64])
def test_every_probe_path(b2, typ):
    """negative keys over 10x the rows (the q3 density): INNER maps with and without a selection vector, the filter inside
    the probe, RIGHT OUTER tracked, a nullable probe key column, and LEFT OUTER / SEMI / ANTI / FULL OUTER through the hash
    table the first such probe builds"""
    rng = np.random.default_rng(int(typ))
    nb, span = 300_000, 3_000_000
    lo = -1_234_567
    bkeys = lo + np.r_[0, span - 1, 1 + rng.choice(span - 2, nb - 2, replace=False)]   # both ends of the span present
    build_cols = [typed(bkeys, typ)]
    ht, layout = build(b2, build_cols)
    assert layout == "direct"
    pk = edge_probe_keys(rng, bkeys, typ)
    pr = [typed(pk, typ)]
    pt = to_table(b2, pr)
    want = join_maps_all(build_cols, pr, False)
    got, names = probe(b2, ht, pt, INNER)
    assert_maps(INNER, got, want[INNER], "inner")
    assert ONE_KEY in names and HASH_BUILD not in names, names
    sel = np.unique(np.r_[np.flatnonzero(rng.random(len(pk)) < 0.3), len(pk) - 1]).astype(np.int32)
    got, names = probe(b2, ht, pt, INNER, b2.Column.from_numpy(sel))
    wl, wr = join_maps(build_cols, [O.OCol(pr[0].values[sel], pr[0].valid[sel], pr[0].typ)], INNER)
    assert_maps(INNER, got, (sel.astype(np.int64)[wl], wr), "inner, selection vector")
    assert ONE_KEY in names and HASH_BUILD not in names, names
    got, names = probe(b2, ht, pt, RIGHT_OUTER)
    assert_right_outer(got, right_outer_maps(build_cols, pr), "right outer")
    assert "join_probe_distinct1_track_kernel" in names and HASH_BUILD not in names, names
    # the filter inside the probe (maps) on a stream batch of [key, d]
    d = rng.integers(0, 100, len(pk)).astype(np.int32)
    st = b2.Table.from_columns([to_table(b2, pr).column(0), b2.Column.from_numpy(d)])
    (lm, rm, npass), names = profiled(b2, lambda: ht.probe_filter(st, 0, b2.Program([b2.col(1, b2.INT32, nullable=False) >= b2.lit(40, b2.INT32)])))
    keep = np.flatnonzero(d >= 40)
    wl, wr = join_maps(build_cols, [O.OCol(pr[0].values[keep], pr[0].valid[keep], pr[0].typ)], INNER)
    assert npass == len(keep) and "join_filter_probe_kernel" in names and HASH_BUILD not in names, names
    assert_maps(INNER, (lm.to_numpy()[0].astype(np.int64), rm.to_numpy()[0].astype(np.int64)), (keep[wl], wr), "filter probe")
    # a nullable probe key column and the kinds without a direct probe: the hash table is built once, on the first of them
    pv = rng.random(len(pk)) > 0.1
    prn = [O.OCol(pr[0].values, pv, pr[0].typ)]
    got, names = probe(b2, ht, to_table(b2, prn), INNER)
    assert_maps(INNER, got, join_maps(build_cols, prn, INNER), "nullable probe keys")
    assert HASH_BUILD in names and ONE_KEY not in names, names
    for kind in (LEFT_OUTER, SEMI, ANTI, FULL_OUTER):
        got, names = probe(b2, ht, pt, kind)
        assert_maps(kind, got, want[kind], kind)
        assert HASH_BUILD not in names, (kind, names)
    got, names = probe(b2, ht, pt, INNER)
    assert_maps(INNER, got, want[INNER], "inner after the hash table")
    assert ONE_KEY in names, names


def test_first_hash_probes_from_many_threads(b2):
    """task threads share one direct table, each on its own stream: several take its first SEMI / LEFT OUTER / ANTI probe at
    once (each would build the hash table) while others probe it directly.  The hash table is built once per table and every
    thread's maps equal the reference"""
    import threading
    rng = np.random.default_rng(31)
    nb, nthreads, rounds = 2_000_000, 8, 3
    kinds = [SEMI, LEFT_OUTER, ANTI, INNER, SEMI, LEFT_OUTER, FULL_OUTER, INNER]
    bkeys = rng.permutation(10 * nb)[:nb].astype(np.int64) - 12345
    build_cols = [ocol(bkeys, O.INT64)]
    pr = [ocol(rng.integers(-20000, 10 * nb, 500_000), O.INT64)]
    want = join_maps_all(build_cols, pr, False)
    pt = to_table(b2, pr)
    b2.profile_enable(True)
    try:
        for r in range(rounds):
            ht = b2.JoinHashTable(to_table(b2, build_cols))
            out, errors = [None] * nthreads, []
            gate = threading.Barrier(nthreads)

            def run(i):
                try:
                    gate.wait()
                    lm, rm = ht.probe(pt, kinds[i])
                    out[i] = (lm.to_numpy()[0].astype(np.int64), None if rm is None else rm.to_numpy()[0].astype(np.int64))
                except Exception as e:   # noqa: BLE001 - reported below
                    errors.append(e)
            th = [threading.Thread(target=run, args=(i,)) for i in range(nthreads)]
            [t.start() for t in th]
            [t.join() for t in th]
            assert not errors, errors
            for i in range(nthreads):
                assert_maps(kinds[i], out[i], want[kinds[i]], (r, i, kinds[i]))
            del ht
        launches = {k["name"]: k["launches"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    assert launches.get(DIRECT_BUILD) == rounds and launches.get(HASH_BUILD) == rounds, launches
    assert launches.get(ONE_KEY, 0) >= 2 * rounds, launches


# ---- 2. the gate ----------------------------------------------------------------------------------------------------------------
def _gate_case(b2, rng, n, span, base, layout):
    keys = base + np.r_[0, span - 1, 1 + rng.choice(span - 2, n - 2, replace=False)]
    cols = [ocol(keys.astype(np.int64), O.INT64)]
    ht, got = build(b2, cols)
    assert got == layout, (n, span, got)
    pk = np.r_[rng.choice(keys, 2 * n), base + rng.integers(-5, span + 5, n)]
    pr = [ocol(pk, O.INT64)]
    res, names = probe(b2, ht, to_table(b2, pr), INNER)
    assert_maps(INNER, res, join_maps(cols, pr, INNER), (n, span))


@pytest.mark.parametrize("n", [1000, 100_003])
def test_gate_density(b2, n):
    """R = 64 x rows is direct, 64 x rows + 1 is not"""
    rng = np.random.default_rng(n)
    _gate_case(b2, rng, n, 64 * n, -17, "direct")
    _gate_case(b2, rng, n, 64 * n + 1, -17, "hash")


def test_gate_span(b2):
    """R = 2^28 is direct, 2^28 + 1 is not (with enough rows that the density allows both)"""
    rng = np.random.default_rng(28)
    _gate_case(b2, rng, 1 << 22, 1 << 28, 5, "direct")
    _gate_case(b2, rng, (1 << 22) + 1, (1 << 28) + 1, 5, "hash")


def test_int64_extremes(b2):
    """build keys at INT64 min and max: the span does not fit 64 bits; the hash table, and every key found"""
    keys = np.array([-2**63, 2**63 - 1, 0, -1, 1], np.int64)
    cols = [ocol(keys, O.INT64)]
    ht, layout = build(b2, cols)
    assert layout == "hash"
    pr = [ocol(np.r_[keys, -2**63 + 1, 2**63 - 2, 2], O.INT64)]
    got, _ = probe(b2, ht, to_table(b2, pr), INNER)
    assert_maps(INNER, got, join_maps(cols, pr, INNER))
    # the same keys next to one extreme: direct, and the wrapping offsets of far keys miss
    for base in (-2**63, 2**63 - 100):
        keys = base + np.arange(0, 100, 3, dtype=np.int64)
        cols = [ocol(keys, O.INT64)]
        ht, layout = build(b2, cols)
        assert layout == "direct"
        pr = [ocol(np.r_[keys, base + np.arange(100), -2**63, 2**63 - 1, 0, -base - 1], O.INT64)]
        got, _ = probe(b2, ht, to_table(b2, pr), INNER)
        assert_maps(INNER, got, join_maps(cols, pr, INNER), base)


# ---- 3. key edges ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", [O.INT32, O.DATE32, O.DECIMAL32, O.TIMESTAMP_US])
def test_key_types_at_their_extremes(b2, typ):
    """a dense key range at each end of the type, and probe keys at the type's extremes"""
    rng = np.random.default_rng(int(typ) + 100)
    tmin, tmax = TYPE_RANGE[typ]
    for lo in (tmin, tmax - 999, -500):
        keys = np.array([lo + int(x) for x in rng.choice(1000, 300, replace=False)], np.int64)
        cols = [typed(keys, typ)]
        ht, layout = build(b2, cols)
        assert layout == "direct"
        pr = [typed(edge_probe_keys(rng, keys, typ), typ)]
        got, _ = probe(b2, ht, to_table(b2, pr), INNER)
        assert_maps(INNER, got, join_maps(cols, pr, INNER), lo)


def test_single_row_build(b2):
    for key in (-7, 0, 2**40):
        cols = [ocol(np.array([key], np.int64), O.INT64)]
        ht, layout = build(b2, cols)
        assert layout == "direct"
        pr = [ocol(np.array([key, key - 1, key + 1, key, -2**63, 2**63 - 1], np.int64), O.INT64)]
        got, _ = probe(b2, ht, to_table(b2, pr), INNER)
        assert sorted(zip(*got)) == [(0, 0), (3, 0)]
        got, _ = probe(b2, ht, to_table(b2, pr), RIGHT_OUTER)
        assert_right_outer(got, right_outer_maps(cols, pr))


def test_null_build_keys(b2):
    """NULL build keys are never matched, whatever bytes lie under them; an all-NULL build side takes the hash table"""
    rng = np.random.default_rng(4)
    n = 50_000
    keys = rng.permutation(4 * n)[:n].astype(np.int64) - 1000
    valid = rng.random(n) > 0.2
    keys[~valid] = keys[valid][: (~valid).sum()]          # a NULL row hides a present key
    cols = [ocol(keys, O.INT64, valid)]
    ht, layout = build(b2, cols)
    assert layout == "direct"
    pr = [ocol(np.r_[keys, rng.integers(-2000, 4 * n, n)], O.INT64)]
    pt = to_table(b2, pr)
    want = join_maps_all(cols, pr, False)
    for kind in (INNER, RIGHT_OUTER):
        got, _ = probe(b2, ht, pt, kind)
        if kind == INNER:
            assert_maps(INNER, got, want[INNER])
            assert not np.isin(got[1], np.flatnonzero(~valid)).any()
        else:
            assert_right_outer(got, right_outer_maps(cols, pr))
    for kind in (LEFT_OUTER, SEMI, ANTI, FULL_OUTER):
        got, _ = probe(b2, ht, pt, kind)
        assert_maps(kind, got, want[kind], kind)
    cols = [ocol(keys, O.INT64, np.zeros(n, bool))]
    ht, layout = build(b2, cols)
    assert layout == "hash"
    got, _ = probe(b2, ht, pt, INNER)
    assert len(got[0]) == 0


def test_duplicate_key_takes_count_and_write(b2):
    rng = np.random.default_rng(6)
    n = 20_000
    keys = rng.permutation(3 * n)[:n].astype(np.int64)
    keys[-1] = keys[n // 2]
    cols = [ocol(keys, O.INT64)]
    ht, layout = build(b2, cols)
    assert layout == "hash"
    pr = [ocol(rng.integers(-10, 3 * n + 10, 4 * n), O.INT64)]
    got, names = probe(b2, ht, to_table(b2, pr), INNER)
    assert_maps(INNER, got, join_maps(cols, pr, INNER))
    assert {"join_probe_count_kernel", "join_probe_write_kernel"} <= names, names


# ---- 4. the exec: the emitting probe and sub-partitioned joins ------------------------------------------------------------------
def _exec_join(b2, E, batches, bt, pred, **kw):
    flt = E.GpuFilterExec(pred, E.GpuBatchSource(batches))
    j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, flt, E.GpuBatchSource([bt]), stream_out=[0, 2], build_out=[1, 2], **kw)
    out, names = profiled(b2, lambda: [t.to_rows() for t in j])
    return sorted(r for rows in out for r in rows), names, j


@pytest.mark.parametrize("kt", [np.int64, np.int32])
def test_emitting_probe(b2, monkeypatch, kt):
    """GpuFilterExec under GpuShuffledHashJoinExec: the first batch through the maps, the others written by the probe from a
    payload packed in rank order; the same rows as the reference and as the hash table"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(12)
    nbatch, per, dom = 4, 200_003, 2_000_000
    skey = rng.integers(-1000, dom + 1000, nbatch * per).astype(kt)
    sdate = rng.integers(8000, 11000, nbatch * per).astype(np.int32)
    sval = rng.integers(0, 1 << 40, nbatch * per).astype(np.int64)
    bkey = rng.permutation(dom)[: dom // 5].astype(kt)
    bval = (bkey.astype(np.int64) * 3 + 1)
    bpay = rng.integers(-2**31, 2**31, len(bkey)).astype(np.int32)
    batches = [b2.Table.from_columns([b2.Column.from_numpy(skey[i * per:(i + 1) * per]), b2.Column.from_numpy(sdate[i * per:(i + 1) * per], dtype=b2.DATE32),
                                      b2.Column.from_numpy(sval[i * per:(i + 1) * per])]) for i in range(nbatch)]
    bt = b2.Table.from_columns([b2.Column.from_numpy(bkey), b2.Column.from_numpy(bval), b2.Column.from_numpy(bpay)])
    pred = b2.Program([b2.col(1, b2.DATE32, nullable=False) > b2.lit(9204, b2.DATE32)])
    keep = sdate > 9204
    pos = {int(k): i for i, k in enumerate(bkey)}
    want = sorted((int(k), int(v), int(bval[pos[int(k)]]), int(bpay[pos[int(k)]])) for k, v, ok in zip(skey, sval, keep) if ok and int(k) in pos)
    got, names, j = _exec_join(b2, E, batches, bt, pred)
    assert got == want
    assert DIRECT_BUILD in names and HASH_BUILD not in names and "join_pack_payload_kernel" in names, names
    assert j.emit_stats["emitted"] == nbatch - 1, j.emit_stats
    monkeypatch.setenv("B2_JOIN_NO_DIRECT", "1")
    got, names, j = _exec_join(b2, E, batches, bt, pred)
    assert got == want and HASH_BUILD in names and DIRECT_BUILD not in names, names
    assert j.emit_stats["emitted"] == nbatch - 1, j.emit_stats


def test_sub_partitioned_join(b2):
    """a build side over the target: hash buckets of dense keys keep their span and lose density, and each bucket's build
    chooses its own layout (16 buckets of keys over 2x the rows: 32x per bucket, direct; over 8x: 128x, hash)"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(21)
    for spread, layout in ((2, DIRECT_BUILD), (8, HASH_BUILD)):
        nb, ns = 400_000, 600_000
        bkey = rng.permutation(spread * nb)[:nb].astype(np.int64)
        bval = rng.integers(0, 1 << 30, nb).astype(np.int64)
        skey = rng.integers(-5, spread * nb + 5, ns).astype(np.int64)
        sf = rng.integers(0, 1000, ns).astype(np.int32)
        stream = [b2.Table.from_columns([b2.Column.from_numpy(skey[i::3]), b2.Column.from_numpy(sf[i::3])]) for i in range(3)]
        bt = [b2.Table.from_columns([b2.Column.from_numpy(bkey[i::2]), b2.Column.from_numpy(bval[i::2])]) for i in range(2)]
        j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, E.GpuBatchSource(stream), E.GpuBatchSource(bt), stream_out=[0, 1], build_out=[1],
                                      target_bytes=nb * 6 // 5, num_sub_partitions=16)   # 16 B per build row: one bucket per build
        b2.profile_enable(True)
        try:
            out = [t.to_rows() for t in j]
            launches = {k["name"]: k["launches"] for k in b2.profile_report()}
        finally:
            b2.profile_enable(False)
        assert j.sub_partition_stats["buckets"] == 16, j.sub_partition_stats
        # every build (each one starts with the range reduction) took the layout, none the other
        builds = launches.get("join_key_range_kernel", 0)
        other = HASH_BUILD if layout == DIRECT_BUILD else DIRECT_BUILD
        assert builds >= 8 and launches.get(layout) == builds and other not in launches, launches
        lut = dict(zip(bkey.tolist(), bval.tolist()))
        order = np.r_[np.arange(0, ns, 3), np.arange(1, ns, 3), np.arange(2, ns, 3)]
        want = sorted((int(k), int(f), lut[int(k)]) for k, f in zip(skey[order], sf[order]) if int(k) in lut)
        assert sorted(r for rows in out for r in rows) == want


# ---- 5. the hash table at the shapes the direct layout now takes ----------------------------------------------------------------
HASH_SUITES = ["tests/test_join_paths_gpu.py", "tests/test_join_filter_probe_gpu.py", "tests/test_join_emit_gpu.py", "tests/test_build_outer_join_gpu.py",
               "tests/test_sub_partition_join_gpu.py"]


def test_join_suites_on_the_hash_table_in_a_child_process():
    """the join suites again with B2_JOIN_NO_DIRECT=1: their dense distinct keys, which now build direct tables, keep the hash
    table's coverage"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    e = dict(os.environ)
    e["B2_JOIN_NO_DIRECT"] = "1"
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider"] + HASH_SUITES, cwd=root, env=e, capture_output=True,
                       text=True, timeout=3600)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
