"""Outer joins that preserve the build side: JOIN_RIGHT_OUTER through every probe path of join.cu, the JoinTracker across
probe batches, and GpuShuffledHashJoinExec with RIGHT OUTER (and FULL OUTER with a condition) over batches, filters,
pruning, memory limits and sub-partitioning, against exact references.

RIGHT OUTER's reference maps are the FULL OUTER rows of join_maps that carry a build row: the inner pairs, then
(INT32_MIN, b) for every build row b no probe row matched.  Each primitive probe asserts from the kernel timings which
tracking probe kernel ran."""
import gc

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from tests.test_join_paths_gpu import (BLOOM_ROWS, INT32_MIN, NPROBE, expected_kernels, join_maps, join_maps_all, key_of,
                                       matrix_input, ocol, selections, take, to_table)
from tests.test_out_of_core_sort_gpu import KEY_TYPES, _key
from tests.test_sub_partition_join_gpu import _assert_join, _build_bytes, _sides, long_pids

pytestmark = pytest.mark.gpu

INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER, RIGHT_OUTER = range(6)
ERR_INVALID, ERR_UNSUPPORTED = 1, 5
TRACK_KERNELS = {"join_probe_distinct1_track_kernel", "join_probe_distinct_track_kernel", "join_probe_write_track_kernel",
                 "join_filter_probe_track_kernel"}
PROBE_KERNELS = {"join_probe_distinct1_kernel", "join_probe_distinct_kernel", "join_probe_count_kernel", "join_probe_write_kernel",
                 "join_filter_probe_kernel"} | TRACK_KERNELS


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


# ---- references -------------------------------------------------------------------------------------------------------------
def remap(m, rows):
    """map entries m (INT32_MIN = none) through rows"""
    out = np.full(len(m), INT32_MIN, np.int64)
    out[m >= 0] = np.asarray(rows, np.int64)[m[m >= 0]]
    return out


def right_outer_maps(build, probe_cols, nulls_equal=False):
    fl, fr = join_maps_all(build, probe_cols, nulls_equal, [FULL_OUTER])[FULL_OUTER]
    keep = fr != INT32_MIN
    return fl[keep], fr[keep]


def expected_track_kernels(build, probe_cols, nulls_equal, n, inner_total, probe_buffer=None):
    """RIGHT OUTER probes INNER with the tracking variant of the kernel INNER takes (the count kernel writes no pairs)"""
    ks = expected_kernels(build, probe_cols, INNER, nulls_equal, n, inner_total, probe_buffer)
    return {k if k == "join_probe_count_kernel" else k.replace("_kernel", "_track_kernel") for k in ks}


def probe(b2, ht, probe_table, kind, selection=None):
    b2.profile_enable(True)
    try:
        lm, rm = ht.probe(probe_table, kind, selection=selection)
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return (lm.to_numpy()[0].astype(np.int64), rm.to_numpy()[0].astype(np.int64)), names & PROBE_KERNELS


def assert_right_outer(got, want, what=""):
    """same pairs; the unmatched build rows come last, ascending"""
    (gl, gr), (wl, wr) = got, want
    assert len(gl) == len(wl), (what, len(gl), len(wl))
    o, p = np.lexsort((gr, gl)), np.lexsort((wr, wl))
    assert np.array_equal(gl[o], wl[p]) and np.array_equal(gr[o], wr[p]), what
    tail = np.flatnonzero(gl == INT32_MIN)
    assert np.array_equal(tail, np.arange(len(gl) - len(tail), len(gl))), what
    assert np.all(np.diff(gr[tail]) > 0), what


def check_right_outer(b2, build, probe_cols, nulls_equal=(False, True), what=""):
    pt = to_table(b2, probe_cols)
    for ne in nulls_equal:
        ht = b2.JoinHashTable(to_table(b2, build), ne)
        want = right_outer_maps(build, probe_cols, ne)
        got, ran = probe(b2, ht, pt, RIGHT_OUTER)
        assert_right_outer(got, want, (what, ne))
        inner = int((want[0] != INT32_MIN).sum())
        assert ran == expected_track_kernels(build, probe_cols, ne, len(probe_cols[0].values), inner), (what, ne, ran)


# ---- 1. the primitive's maps ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb", [100_000, BLOOM_ROWS, BLOOM_ROWS + 1], ids=["bloom_off", "bloom_2^18", "bloom_2^18+1"])
@pytest.mark.parametrize("dup", [False, True], ids=["distinct", "duplicates"])
@pytest.mark.parametrize("layout", ["packed", "generic"])
def test_right_outer_path_matrix(b2, monkeypatch, layout, dup, nb):
    """packed and generic tables, distinct and duplicate build sides, the Bloom filter off and on, through no selection
    vector, an empty one, one of every row and a sparse one"""
    monkeypatch.delenv("B2_JOIN_NO_BLOOM", raising=False)
    monkeypatch.delenv("B2_JOIN_NO_FAST_PROBE", raising=False)
    build, pr = matrix_input(layout, dup, nb, seed=nb + 7 * dup + (layout == "generic"))
    ht = b2.JoinHashTable(to_table(b2, build))
    pt = to_table(b2, pr)
    rng = np.random.default_rng(12)
    for sname, sel in selections(rng, NPROBE).items():
        sub = pr if sel is None else take(pr, sel)
        wl, wr = right_outer_maps(build, sub)
        if sel is not None:                     # the left map carries original row ids
            wl = remap(wl, sel)
        got, ran = probe(b2, ht, pt, RIGHT_OUTER, None if sel is None else b2.Column.from_numpy(sel))
        assert_right_outer(got, (wl, wr), sname)
        inner = int((wl != INT32_MIN).sum())
        assert ran == expected_track_kernels(build, sub, False, len(sub[0].values), inner), (sname, ran)
        if sname == "none":
            assert 0 < inner and 0 < len(wl) - inner < nb     # some build rows matched, some did not


@pytest.mark.parametrize("typ", KEY_TYPES, ids=lambda t: str(t[0]))
def test_right_outer_key_types(b2, typ):
    """one key of every type with NULL keys on both sides, under nulls_equal 0 and 1; a distinct build side too"""
    rng = np.random.default_rng(30 + typ[0])
    base = _key(rng, typ, 400, False, maxlen=6)
    build = take([base], rng.integers(0, 400, 300))
    pr = take([base], rng.integers(0, 400, 2000))
    build[0].valid = rng.random(300) > 0.15
    pr[0].valid = rng.random(2000) > 0.15
    check_right_outer(b2, build, pr, what=typ)
    vals = build[0].values
    first = np.sort(np.unique(np.asarray([repr(v) for v in vals], dtype=object), return_index=True)[1])
    distinct = take(build, first)
    distinct[0].valid[:] = True
    check_right_outer(b2, distinct, pr, what=(typ, "distinct"))


@pytest.mark.parametrize("nb", [0, 1, 31, 32, 33])
def test_right_outer_sizes(b2, nb):
    rng = np.random.default_rng(nb)
    for npr in (0, 1, 33):
        for kt in (O.INT64, O.STRING):
            def keys(n):
                v = rng.integers(0, 20, n)
                return [ocol(v.astype(np.int64), O.INT64) if kt == O.INT64 else ocol(np.array([b"k%d" % x for x in v], dtype=object), O.STRING)]
            build, pr = keys(nb), keys(npr)
            check_right_outer(b2, build, pr, what=(kt, nb, npr))
            if nb:
                first = np.sort(np.unique(build[0].values, return_index=True)[1])
                check_right_outer(b2, take(build, first), pr, what=(kt, nb, npr, "distinct"))


def test_full_outer_maps_unchanged(b2):
    """the single-batch FULL OUTER primitive (now marked through the tracker) against join_maps, unmatched rows ascending"""
    for nb in (0, 33, 70_000, BLOOM_ROWS + 1):
        for dup in (False, True):
            build, pr = matrix_input("packed", dup, max(nb, 1), seed=nb + dup)
            build = take(build, np.arange(nb))
            ht = b2.JoinHashTable(to_table(b2, build))
            (gl, gr), _ = probe(b2, ht, to_table(b2, pr), FULL_OUTER)
            wl, wr = join_maps(build, pr, FULL_OUTER)
            o, p = np.lexsort((gr, gl)), np.lexsort((wr, wl))
            assert np.array_equal(gl[o], wl[p]) and np.array_equal(gr[o], wr[p]), (nb, dup)
            tail = gr[gl == INT32_MIN]
            assert np.array_equal(tail, wr[wl == INT32_MIN]), (nb, dup)     # ascending, as the reference


# ---- 2. the tracker across batches ------------------------------------------------------------------------------------------
def test_tracker_across_batches(b2):
    rng = np.random.default_rng(21)
    nb = 200_003                                   # four tiles of 65536 rows, a tail word of 3 bits
    for layout, dup in (("packed", False), ("generic", False), ("packed", True)):
        build, _ = matrix_input(layout, dup, nb, seed=5)
        ht = b2.JoinHashTable(to_table(b2, build))
        tr = b2.JoinTracker(ht)
        assert np.array_equal(tr.unmatched().to_numpy()[0], np.arange(nb))
        hit = np.zeros(nb, bool)
        for i in range(3):
            bk = build[0].values
            pk = np.where(rng.random(50_000) < 0.4, bk[rng.integers(0, nb, 50_000)], key_of(10**7 + rng.integers(0, 10**6, 50_000)))
            pr = [ocol(pk, O.INT64)] if layout == "packed" else [ocol(pk, O.INT64), ocol((rng.integers(0, 2001, 50_000) - 1000).astype(np.int32), O.INT32)]
            if layout == "generic":       # match the second key where the first one does
                pos = {int(v): j for j, v in enumerate(bk)}
                at = np.array([pos.get(int(v), -1) for v in pk])
                pr[1].values[at >= 0] = build[1].values[at[at >= 0]]
            kind = INNER if i != 1 else LEFT_OUTER
            pt = to_table(b2, pr)
            lm, rm = tr.probe(ht, pt, kind)
            gl, gr = lm.to_numpy()[0].astype(np.int64), rm.to_numpy()[0].astype(np.int64)
            wl, wr = join_maps(build, pr, kind)
            o, p = np.lexsort((gr, gl)), np.lexsort((wr, wl))
            assert np.array_equal(gl[o], wl[p]) and np.array_equal(gr[o], wr[p]), (layout, i)
            hit[wr[wr >= 0]] = True
            assert np.array_equal(tr.unmatched().to_numpy()[0], np.flatnonzero(~hit)), (layout, i)   # bits = union of the right maps
            tr.probe(ht, pt, kind)                                                                      # the same batch again
            assert np.array_equal(tr.unmatched().to_numpy()[0], np.flatnonzero(~hit)), (layout, i)
        sel = np.flatnonzero(rng.random(50_000) < 0.3).astype(np.int32)
        tr.probe(ht, pt, INNER, selection=b2.Column.from_numpy(sel))
        assert np.array_equal(tr.unmatched().to_numpy()[0], np.flatnonzero(~hit))


def test_tracker_mark_and_errors(b2):
    rng = np.random.default_rng(22)
    for nb in (1, 31, 32, 33, 65_536, 65_537, 100_000):
        ht = b2.JoinHashTable(to_table(b2, [ocol(key_of(np.arange(nb)), O.INT64)]))
        tr = b2.JoinTracker(ht)
        rmap = rng.integers(0, nb, 3000).astype(np.int32)
        rmap[rng.random(3000) < 0.1] = INT32_MIN
        passed = rng.integers(0, 2, 3000).astype(np.int8)
        pvalid = rng.random(3000) > 0.2
        tr.mark(b2.Column.from_numpy(rmap), b2.Column.from_numpy(passed, dtype=b2.BOOL8, valid=pvalid))
        hit = np.zeros(nb, bool)
        ok = (rmap >= 0) & (passed != 0) & pvalid
        hit[rmap[ok]] = True
        assert np.array_equal(tr.unmatched().to_numpy()[0], np.flatnonzero(~hit)), nb
        tr.mark(b2.Column.from_numpy(rmap))                      # no mask: every non-negative entry
        hit[rmap[rmap >= 0]] = True
        assert np.array_equal(tr.unmatched().to_numpy()[0], np.flatnonzero(~hit)), nb
        tr.mark(b2.Column.from_numpy(np.arange(nb, dtype=np.int32)))
        assert len(tr.unmatched().to_numpy()[0]) == 0
        with pytest.raises(b2.B2Error) as e:
            tr.mark(b2.Column.from_numpy(np.array([0, nb], np.int32)))
        assert e.value.code == ERR_INVALID
    other = b2.JoinHashTable(to_table(b2, [ocol(key_of(np.arange(10)), O.INT64)]))
    pt = to_table(b2, [ocol(key_of(np.arange(5)), O.INT64)])
    with pytest.raises(b2.B2Error) as e:
        tr.probe(other, pt, INNER)
    assert e.value.code == ERR_INVALID
    for kind in (SEMI, ANTI, FULL_OUTER, RIGHT_OUTER):
        with pytest.raises(b2.B2Error) as e:
            tr.probe(ht, pt, kind)
        assert e.value.code == ERR_INVALID


# ---- 3. the exec ----------------------------------------------------------------------------------------------------------------
def _reference(stream, build, keep, kind, nulls_equal, cond, so, bo):
    """RIGHT OUTER: the (conditional) inner pairs, then every build row without one; FULL OUTER adds every stream row
    without one.  cond: f >= bid over the pairs"""
    rows = np.flatnonzero(keep)
    st = take(stream, rows)
    il, ir = join_maps(build[:1], st[:1], INNER, nulls_equal)
    if cond:
        ok = st[1].values[il] >= build[1].values[ir]
        il, ir = il[ok], ir[ok]
    hitb = np.zeros(len(build[0].values), bool)
    hitb[ir] = True
    unb = np.flatnonzero(~hitb)
    lm, rm = np.r_[il, np.full(len(unb), INT32_MIN)], np.r_[ir, unb]
    if kind == FULL_OUTER:
        hits = np.zeros(len(rows), bool)
        hits[il] = True
        lonely = np.flatnonzero(~hits)
        lm, rm = np.r_[lm, lonely], np.r_[rm, np.full(len(lonely), INT32_MIN)]
    lm = remap(lm, rows)
    return R.gather([stream[c] for c in so], lm, True) + R.gather([build[c] for c in bo], rm, True)


FILTERS = {
    "none": None,
    "simple": lambda b2: b2.col(1, b2.INT32, nullable=False) >= b2.lit(500, b2.INT32),
    "like": lambda b2: b2.col(5, b2.STRING).like("%1%"),
}


def _filter_keep(stream, name):
    if name == "simple":
        return stream[1].values >= 500
    if name == "like":
        return np.array([v is not None and ok and b"1" in v for v, ok in zip(stream[5].values, stream[5].valid)])
    return np.ones(len(stream[0].values), bool)


def run_exec(b2, sides, kind, filt, prune, nulls_equal, cond, target=None, nparts=16, ids=(2, 1), names_out=None):
    from spark_rapids_b200 import execs as E
    stream, build, sbatches, bbatches = sides
    gc.collect()
    b2.sync()
    base = b2.device_bytes_in_use()
    src = E.GpuBatchSource([to_table(b2, s) for s in sbatches])
    keep = _filter_keep(stream, filt)
    if filt != "none":
        src = E.GpuFilterExec(FILTERS[filt](b2), src)
    so, bo = ([2, 0, 5, 6, 3], [1, 3, 4, 2]) if prune else (list(range(len(stream))), list(range(len(build))))
    kw = dict(stream_out=so, build_out=bo) if prune else {}
    if cond:
        kw["condition"] = b2.col(1, b2.INT32, nullable=False) >= b2.col(len(stream) + 1, b2.INT32, nullable=False)
    if target is not None:
        kw.update(target_bytes=target, num_sub_partitions=nparts)
    j = E.GpuShuffledHashJoinExec([0], [0], kind, src, E.GpuBatchSource([to_table(b2, b) for b in bbatches]), nulls_equal=nulls_equal, **kw)
    b2.profile_enable(True)
    try:
        outs = list(j)
        if names_out is not None:
            names_out |= {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    out = b2.concat(outs) if len(outs) > 1 else outs[0]
    want = _reference(stream, build, keep, kind, nulls_equal, cond, so, bo)
    _assert_join(out, want, kind, so.index(ids[0]), len(so) + bo.index(ids[1]))
    assert j.metrics["numOutputRows"] == out.num_rows and j.metrics["numOutputBatches"] == len(outs)
    stats = j.sub_partition_stats
    del outs, out, j, src
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base
    return stats


@pytest.mark.parametrize("prune", [False, True], ids=["all_columns", "pruned"])
@pytest.mark.parametrize("filt", ["none", "simple", "like"])
@pytest.mark.parametrize("kind,cond", [(RIGHT_OUTER, False), (RIGHT_OUTER, True), (FULL_OUTER, True)], ids=["right", "right_cond", "full_cond"])
def test_exec(b2, kind, cond, filt, prune):
    """multi-batch stream (one batch empty, the filter passes no row of the last) and build sides (one with NULL keys)"""
    rng = np.random.default_rng(40 + kind + 2 * cond)
    sides = _sides(rng)
    for ne in (False, True):
        names = set()
        run_exec(b2, sides, kind, filt, prune, ne, cond, names_out=names)
        if not cond:
            assert names & TRACK_KERNELS, names
        else:
            assert "tracker_mark_kernel" in names, names


def test_exec_filter_inside_the_probe(b2, monkeypatch):
    """RIGHT OUTER, distinct build side on one INT64 key, a simple filter below and a stream batch of >= 2^16 rows: the
    tracking variant of join_filter_probe_kernel; the same rows through the selection-vector path"""
    rng = np.random.default_rng(44)
    stream, build, sbatches, bbatches = _sides(rng, sizes=((1 << 16) + 100, 0, 3000), stream_nulls=0)
    bk = np.flatnonzero(build[0].valid)                       # distinct, NOT NULL build keys
    sides = (stream, take(build, bk), sbatches, [take(build, bk)])
    names = set()
    run_exec(b2, sides, RIGHT_OUTER, "simple", True, False, False, names_out=names)
    assert "join_filter_probe_track_kernel" in names, names
    monkeypatch.setenv("B2_JOIN_NO_FAST_PROBE", "1")
    names = set()
    run_exec(b2, sides, RIGHT_OUTER, "simple", True, False, False, names_out=names)
    assert "join_probe_distinct_track_kernel" in names and "join_filter_probe_track_kernel" not in names, names


def test_exec_edges(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(45)
    stream, build, sbatches, bbatches = _sides(rng)
    for kind, cond in ((RIGHT_OUTER, None), (FULL_OUTER, b2.col(1, b2.INT32, nullable=False) >= b2.col(8, b2.INT32, nullable=False))):
        j = E.GpuShuffledHashJoinExec([0], [0], kind, E.GpuBatchSource([]), E.GpuBatchSource([to_table(b2, b) for b in bbatches]), condition=cond)
        with pytest.raises(b2.B2Error) as e:            # no stream batch at all: the stream schema is unknown
            j.collect()
        assert e.value.code == ERR_UNSUPPORTED
        j = E.GpuShuffledHashJoinExec([0], [0], kind, E.GpuBatchSource([to_table(b2, s) for s in sbatches]), E.GpuBatchSource([]), condition=cond)
        with pytest.raises(b2.B2Error) as e:
            j.collect()
        assert e.value.code == ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        E.GpuBroadcastHashJoinExec([0], [0], RIGHT_OUTER, E.GpuBatchSource([]), E.GpuBatchSource([]))
    # only empty stream batches: every build row, NULL on the stream side
    e_s = take(stream, np.arange(0))
    run_exec(b2, (e_s, build, [e_s, e_s], bbatches), RIGHT_OUTER, "none", True, False, False)


# ---- 4. beyond the device, and the retry paths ------------------------------------------------------------------------------
def _host(cols, rows):
    return [[(O.INT64, 0, c[s:s + rows], None) for c in cols] for s in range(0, len(cols[0]), rows)]


@pytest.mark.parametrize("kind", [RIGHT_OUTER, FULL_OUTER], ids=["right", "full_cond"])
def test_beyond_the_allocation_limit(b2, limits, kind):
    """an 8 MiB build side (2^18 rows of four INT64 columns: its hash table takes 8.25 MiB more) and a 96 MiB stream side in
    2 MiB host batches, 32 MiB above the base: finishes without sub-partitioning, one stream batch at a time"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(18)
    rows = 1 << 17
    nb, ns = 2 * rows, 48 * rows
    bk = key_of(rng.permutation(nb))
    sk = np.where(rng.random(ns) < 0.7, bk[rng.integers(0, nb // 2, ns)], key_of(nb + rng.integers(0, nb, ns)))   # half the build rows are hit
    bp, sp = np.arange(nb, dtype=np.int64), np.arange(ns, dtype=np.int64) + 10**12
    gc.collect()
    b2.sync()
    base = b2.device_bytes_in_use()
    b2.set_alloc_limit(base + (32 << 20))
    cond = b2.col(3, b2.INT64, nullable=False) >= b2.lit(nb // 8, b2.INT64) if kind == FULL_OUTER else None
    node = E.GpuShuffledHashJoinExec([0], [0], kind, E.GpuHostBatchSource(_host([sk, sp], rows)),
                                     E.GpuHostBatchSource(_host([bk, bp, bp * 3, bp * 5], rows // 2)), condition=cond)
    gs, gb = [], []
    for t in node:
        s, b = t.column(1).to_numpy(), t.column(3).to_numpy()
        gs.append(np.where(s[1], s[0], -1))
        gb.append(np.where(b[1], b[0], -1))
        del t
    assert node.sub_partition_stats["buckets"] == 0
    got_s, got_b = np.concatenate(gs), np.concatenate(gb)
    assert node.metrics["numOutputRows"] == len(got_s)
    il, ir = join_maps([ocol(bk, O.INT64)], [ocol(sk, O.INT64)], INNER)
    if kind == FULL_OUTER:
        ok = ir >= nb // 8
        il, ir = il[ok], ir[ok]
    hitb = np.zeros(nb, bool)
    hitb[ir] = True
    lm, rm = np.r_[il, np.full(nb - hitb.sum(), INT32_MIN)], np.r_[ir, np.flatnonzero(~hitb)]
    if kind == FULL_OUTER:
        hits = np.zeros(ns, bool)
        hits[il] = True
        lonely = np.flatnonzero(~hits)
        lm, rm = np.r_[lm, lonely], np.r_[rm, np.full(len(lonely), INT32_MIN)]
    ws = np.where(lm >= 0, sp[np.maximum(lm, 0)], -1)
    wb = np.where(rm >= 0, bp[np.maximum(rm, 0)], -1)
    og, ow = np.lexsort((got_b, got_s)), np.lexsort((wb, ws))
    assert np.array_equal(got_s[og], ws[ow]) and np.array_equal(got_b[og], wb[ow])
    del node
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base


def _pull_under(b2, j, headroom):
    """every output batch of j, the limit `headroom` above what is in use before each pull -> rows, number of batches"""
    got, nout = [], 0
    while True:
        b2.sync()
        b2.set_alloc_limit(b2.device_bytes_in_use() + headroom)
        t = j.next()
        b2.set_alloc_limit(0)
        if t is None:
            return got, nout
        got += t.to_rows()
        nout += 1
        del t
        gc.collect()


def test_stream_batch_split_and_retry(b2, limits):
    """one 8 MiB stream batch whose join needs 20 MiB at its peak, 15 MiB allowed: halved and retried, same rows"""
    from spark_rapids_b200 import execs as E
    ns, nb = 1 << 19, 1 << 12
    rng = np.random.default_rng(6)
    st = to_table(b2, [ocol(rng.integers(0, nb // 2, ns).astype(np.int64), O.INT64), ocol(np.arange(ns, dtype=np.int64), O.INT64)])
    bt = to_table(b2, [ocol(np.arange(nb, dtype=np.int64), O.INT64), ocol(np.arange(nb, dtype=np.int64) * 3, O.INT64)])
    exp = sorted(E.GpuShuffledHashJoinExec([0], [0], RIGHT_OUTER, E.GpuBatchSource([st]), E.GpuBatchSource([bt])).collect().to_rows(), key=repr)
    assert len(exp) == ns + nb // 2 and sum(r[0] is None for r in exp) == nb // 2
    s0 = b2.memory_stats()
    j = E.GpuShuffledHashJoinExec([0], [0], RIGHT_OUTER, E.GpuBatchSource([st]), E.GpuBatchSource([bt]))
    got, nout = _pull_under(b2, j, 15 << 20)
    s1 = b2.memory_stats()
    assert s1["splits"] > s0["splits"] and nout >= 3, (s0, s1, nout)
    assert sorted(got, key=repr) == exp


def test_final_batch_split(b2, limits):
    """2^19 unmatched build rows whose final gather needs about 20 MiB, 16 MiB allowed: the id range is halved"""
    from spark_rapids_b200 import execs as E
    nb = 1 << 19
    st = to_table(b2, [ocol(key_of(np.arange(nb, nb + 1000)), O.INT64), ocol(np.arange(1000, dtype=np.int64), O.INT64)])
    bt = to_table(b2, [ocol(key_of(np.arange(nb)), O.INT64), ocol(np.arange(nb, dtype=np.int64), O.INT64)])
    j = E.GpuShuffledHashJoinExec([0], [0], RIGHT_OUTER, E.GpuBatchSource([st]), E.GpuBatchSource([bt]))
    first = j.next()                                      # builds the table and joins the only stream batch: no row matches
    assert first.num_rows == 0
    del first
    gc.collect()
    s0 = b2.memory_stats()
    got, nout = _pull_under(b2, j, 16 << 20)
    s1 = b2.memory_stats()
    assert s1["splits"] > s0["splits"] and nout >= 2, (s0, s1, nout)
    assert j.metrics["numOutputBatches"] == nout + 1 and j.metrics["numOutputRows"] == nb
    assert [r[0] for r in got] == [None] * nb and [r[1] for r in got] == [None] * nb
    assert [r[3] for r in got] == list(range(nb))        # ascending build rows, in order across the batches


# ---- 5. sub-partitioning ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cond", [(RIGHT_OUTER, False), (RIGHT_OUTER, True), (FULL_OUTER, True)], ids=["right", "right_cond", "full_cond"])
def test_sub_partitioned(b2, kind, cond):
    rng = np.random.default_rng(50 + kind + cond)
    sides = _sides(rng)
    bb = _build_bytes(b2, sides[3])
    for filt, prune in (("none", False), ("simple", True)):
        for ne in (False, True):
            st = run_exec(b2, sides, kind, filt, prune, ne, cond, bb // 5, 16)       # several packed buckets
            assert st["buckets"] == 16 and st["repartitioned"] == 0 and st["stream_bytes"] > 0, st
            st = run_exec(b2, sides, kind, filt, prune, ne, cond, int(bb * 0.4), 2)  # each half is over: split again
            assert st["buckets"] == 2 and st["repartitioned"] >= 1, st


def _int_sides(bkeys, skeys):
    stream = [ocol(skeys, O.INT64), ocol(np.arange(len(skeys), dtype=np.int32), O.INT32)]
    build = [ocol(bkeys, O.INT64), ocol(np.arange(len(bkeys), dtype=np.int32), O.INT32)]
    half = len(bkeys) // 2
    return stream, build, [stream], [take(build, np.arange(half)), take(build, np.arange(half, len(bkeys)))]


def test_sub_partitioned_skew_and_lonely_build_buckets(b2):
    rng = np.random.default_rng(51)
    cand = key_of(rng.permutation(400_000))
    pid = long_pids(cand, 16, 100)
    bkeys = np.r_[cand[pid == 5][:12000], cand[pid != 5][:3000]]            # bucket 5 holds 80 % of the build rows
    skeys = np.r_[rng.choice(bkeys, 20000), cand[-5000:]]
    st = run_exec(b2, _int_sides(bkeys, skeys), RIGHT_OUTER, "none", False, False, False, 64 << 10, ids=(1, 1))
    assert st["buckets"] == 16 and st["repartitioned"] == 1, st
    # build rows in every bucket, stream rows in 4 of them: the other 12 pairs have no stream piece and emit all their rows
    bkeys = cand[:8000]
    skeys = np.r_[rng.choice(bkeys[long_pids(bkeys, 16, 100) < 4], 3000), cand[-4000:][long_pids(cand[-4000:], 16, 100) < 4]]
    st = run_exec(b2, _int_sides(bkeys, skeys), RIGHT_OUTER, "none", False, False, False, 16 << 10, ids=(1, 1))
    assert st["buckets"] == 16, st
