"""Join build sides larger than the target (GpuSubPartitionHashJoin): b2_hash_split against the murmur3 oracle, and the
sub-partitioned GpuShuffledHashJoinExec against the exact join reference (join_maps) for every join kind, NULL-key rule,
filter below the stream side, column pruning and non-equi condition, with forced repartitions, skew and a build side (and
for FULL OUTER a stream side) larger than the allocation limit."""
import gc

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_hash as H
from oracle import spark_relational as R
from tests.test_join_paths_gpu import INT32_MIN, _payload, join_maps, key_of, ocol, take, to_table
from tests.test_out_of_core_sort_gpu import KEY_TYPES, _key, _table_bytes

pytestmark = pytest.mark.gpu

INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER = range(5)
KINDS = [INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER]
ERR_OOM = 3
M32 = np.uint64(0xFFFFFFFF)


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


# ---- vectorised murmur3 of INT64 keys (for the large inputs), pinned to the oracle below ---------------------------------------
def _mix_k1(k):
    k = (k * np.uint64(0xCC9E2D51)) & M32
    k = ((k << np.uint64(15)) | (k >> np.uint64(17))) & M32
    return (k * np.uint64(0x1B873593)) & M32


def _mix_h1(h, k):
    h = h ^ k
    h = ((h << np.uint64(13)) | (h >> np.uint64(19))) & M32
    return (h * np.uint64(5) + np.uint64(0xE6546B64)) & M32


def _fmix(h, n):
    h = h ^ np.uint64(n)
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85EBCA6B)) & M32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & M32
    return h ^ (h >> np.uint64(16))


def long_pids(keys, nparts, seed):
    """pmod(murmur3(INT64 key, seed), nparts) as numpy arrays"""
    u = np.asarray(keys, dtype=np.int64).view(np.uint64)
    h = _mix_h1(np.full(len(u), np.uint64(seed)), _mix_k1(u & M32))
    h = _fmix(_mix_h1(h, _mix_k1(u >> np.uint64(32))), 8)
    return h.astype(np.uint32).view(np.int32).astype(np.int64) % nparts


def test_long_pids_match_the_oracle():
    keys = key_of(np.arange(3000))
    for k, seed in [(16, 100), (8, 42), (256, 110)]:
        assert np.array_equal(long_pids(keys, k, seed), H.partition_ids([ocol(keys, O.INT64)], k, seed))


# ---- 1. b2_hash_split --------------------------------------------------------------------------------------------------------
def _assert_cols(t, cols, what=""):
    assert t.num_rows == len(cols[0].values), what
    assert t.num_columns == len(cols), what
    for i, oc in enumerate(cols):
        vals, valid = t.column(i).to_numpy()
        assert np.array_equal(valid, oc.valid), "%s column %d validity" % (what, i)
        if oc.typ[0] in (O.STRING, O.DECIMAL128):
            assert [x for x, v in zip(vals, valid) if v] == [x for x, v in zip(oc.values, oc.valid) if v], "%s column %d" % (what, i)
        else:   # bit for bit (floats included)
            w = np.asarray(vals).dtype.itemsize
            exp = np.asarray(oc.values).astype(vals.dtype)
            assert np.array_equal(vals.view("u%d" % w)[valid], exp.view("u%d" % w)[valid]), "%s column %d" % (what, i)


def _check_split(b2, cols, keys, nparts, seed, sel=None, keep=None, pids=None):
    """b2_hash_split of the table of `cols` against bucket = pmod(murmur3(keys, seed), nparts), rows in input order"""
    t = to_table(b2, cols)
    selc = None if sel is None else b2.Column.from_numpy(np.asarray(sel, np.int32))
    got = b2.hash_split(t, keys, seed, nparts, sel=selc, keep=keep)
    rows = np.arange(len(cols[0].values)) if sel is None else np.asarray(sel, np.int64)
    if pids is None:
        pids = H.partition_ids([take([cols[k]], rows)[0] for k in keys], nparts, seed) if len(rows) else np.zeros(0, np.int32)
    kept = cols if keep is None else [cols[c] for c in keep]
    assert len(got) == nparts
    for p in range(nparts):
        idx = rows[pids == p]
        if len(idx) == 0:
            assert got[p] is None, p
        else:
            _assert_cols(got[p], take(kept, idx), "part %d" % p)


@pytest.mark.parametrize("nkeys", [1, 3])
@pytest.mark.parametrize("nullable", [False, True], ids=["not_null", "nullable"])
@pytest.mark.parametrize("typ", KEY_TYPES, ids=lambda t: str(t[0]))
def test_split_key_types(b2, typ, nullable, nkeys):
    """every join key type; nullable fixed-width payload whose runs cross tile boundaries, strings, keep lists that reorder
    and drop columns"""
    rng = np.random.default_rng(100 * typ[0] + 10 * nullable + nkeys)
    n = 5000
    cols = [_key(rng, typ, n, nullable, maxlen=12), _payload(rng, O.INT32, n, True), _payload(rng, O.STRING, n, True),
            _payload(rng, (O.DECIMAL128, 30, 2), n, True), _payload(rng, O.INT16, n, False)]
    keys = [0] if nkeys == 1 else [0, 4, 2]
    for nparts in (16, 255):
        _check_split(b2, cols, keys, nparts, 100)
        _check_split(b2, cols, keys, nparts, 110, keep=[3, 0, 2])


@pytest.mark.parametrize("nparts", [2, 16, 255, 256])
def test_split_sizes_and_selections(b2, nparts):
    rng = np.random.default_rng(nparts)
    for n in (0, 1, 4095, 4096, 4097):
        cols = [ocol(key_of(rng.integers(0, 50, n)), O.INT64, rng.random(n) > 0.1), _payload(rng, O.INT64, n, True), _payload(rng, O.INT8, n, True),
                _payload(rng, (O.DECIMAL128, 30, 2), n, False), _payload(rng, O.STRING, n, True)]
        sparse = np.unique(np.r_[np.flatnonzero(rng.random(n) < 0.15), max(n - 1, 0)])[: n].astype(np.int32)
        pids = H.partition_ids(cols[:1], nparts, 100) if n else np.zeros(0, np.int32)
        for sel in (None, np.zeros(0, np.int32), np.arange(n, dtype=np.int32), sparse):
            ps = pids if sel is None else pids[sel]
            _check_split(b2, cols, [0], nparts, 100, sel=sel, pids=ps)
            _check_split(b2, cols, [0], nparts, 100, sel=sel, keep=[4, 1], pids=ps)


@pytest.mark.parametrize("nparts", [16, 256])
def test_split_three_million_rows(b2, nparts):
    rng = np.random.default_rng(3)
    n = 3_000_000
    keys = rng.integers(-2**62, 2**62, n)
    cols = [ocol(keys, O.INT64), _payload(rng, O.INT32, n, True), ocol(rng.random(n), O.FLOAT64), _payload(rng, O.INT8, n, False)]
    pids = long_pids(keys, nparts, 100)
    b2.sync()
    b2.profile_enable(True)
    try:
        _check_split(b2, cols, [0], nparts, 100, keep=[1, 2, 0, 3], pids=pids)
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    assert {"hash_split_count_kernel", "hash_split_scatter_kernel"} <= names, names
    sel = np.flatnonzero(rng.random(n) < 0.3).astype(np.int32)
    _check_split(b2, cols, [0], nparts, 100, sel=sel, pids=pids[sel])


# ---- 2. equal keys stay together; 3. no correlation with the exchange ---------------------------------------------------------
SPECIAL_F64 = np.array([0x0, 0x8000000000000000, 0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF],
                       dtype=np.uint64).view(np.float64)


def test_float_specials_share_a_bucket(b2):
    rng = np.random.default_rng(8)
    for dt, vals in [(O.FLOAT64, SPECIAL_F64), (O.FLOAT32, SPECIAL_F64.astype(np.float32))]:
        n = 6000
        v = np.where(rng.random(n) < 0.5, vals[rng.integers(0, len(vals), n)], rng.integers(-3, 3, n)).astype(vals.dtype)
        t = to_table(b2, [ocol(v, dt), ocol(np.arange(n, dtype=np.int32), O.INT32)])
        parts = b2.hash_split(t, [0], 100, 16)
        bucket = np.full(n, -1)
        for p, pt in enumerate(parts):
            if pt is not None:
                bucket[pt.column(1).to_numpy()[0]] = p
        with np.errstate(invalid="ignore"):
            cls = np.where(np.isnan(v), np.nan, np.where(v == 0, 0.0, v))
        for c in np.unique(cls[~np.isnan(cls)]):
            assert len(np.unique(bucket[cls == c])) == 1
        assert len(np.unique(bucket[np.isnan(cls)])) == 1


def test_buckets_do_not_follow_the_exchange(b2):
    """keys that all went to rank 3 of 8 by murmur3 seed 42 still fill all 16 buckets evenly; with seed 42 only 2 would"""
    rng = np.random.default_rng(42)
    cand = rng.integers(-2**62, 2**62, 12_000_000)
    keys = cand[long_pids(cand, 8, 42) == 3][:1_000_000]
    assert len(keys) == 1_000_000
    t = to_table(b2, [ocol(keys, O.INT64)])
    counts = [0 if p is None else p.num_rows for p in b2.hash_split(t, [0], 100, 16)]
    assert min(counts) >= 0.9 * len(keys) / 16 and max(counts) <= 1.1 * len(keys) / 16, counts
    assert sum(p is not None for p in b2.hash_split(t, [0], 42, 16)) == 2


# ---- 4. the join ---------------------------------------------------------------------------------------------------------------
def _sides(rng, key_dt=O.INT64, sizes=(20000, 0, 3000), stream_nulls=0.05):
    """stream: three batches (one empty) of [key, f INT32, sid INT32, i16, i32 nullable, str nullable, dec128];
    build: three batches (one empty), the third with NULL keys and NULL payload, of [key, bid INT32, i8, dec128, str]"""
    bsizes = [3000, 0, 2000]
    ns, nb = sum(sizes), sum(bsizes)
    ids = rng.permutation(4 * nb)[:nb]
    mk = (lambda x: key_of(x)) if key_dt == O.INT64 else (lambda x: (np.asarray(x) % 700 - 350).astype(np.float64) * 0.5)
    bkey = mk(ids)
    if key_dt == O.FLOAT64:   # -0.0 / NaN payloads on both sides
        bkey[:40] = SPECIAL_F64[np.arange(40) % len(SPECIAL_F64)]
    bvalid = np.r_[np.ones(3000, bool), rng.random(2000) > 0.2]
    build = [ocol(bkey, key_dt, bvalid), ocol(np.arange(nb, dtype=np.int32), O.INT32), _payload(rng, O.INT8, nb, False),
             _payload(rng, (O.DECIMAL128, 30, 2), nb, False), _payload(rng, O.STRING, nb, False)]
    for c in build[2:]:
        c.valid[3000:] = rng.random(2000) > 0.3
    skey = mk(np.where(rng.random(ns) < 0.6, rng.choice(ids, ns), 4 * nb + rng.integers(0, 1000, ns)))
    if key_dt == O.FLOAT64:
        skey[:60] = SPECIAL_F64[(np.arange(60) * 5) % len(SPECIAL_F64)]
    svalid = rng.random(ns) >= stream_nulls
    stream = [ocol(skey, key_dt, svalid), ocol(rng.integers(0, 1000, ns).astype(np.int32), O.INT32), ocol(np.arange(ns, dtype=np.int32), O.INT32),
              _payload(rng, O.INT16, ns, False), _payload(rng, O.INT32, ns, True), _payload(rng, O.STRING, ns, True),
              _payload(rng, (O.DECIMAL128, 30, 2), ns, False)]
    bounds = np.cumsum([0] + list(sizes))
    stream[1].values[bounds[2]:] = rng.integers(0, 500, sizes[2])       # the filter passes no row of the last batch
    bb = np.cumsum([0] + bsizes)
    return (stream, build, [take(stream, np.arange(bounds[i], bounds[i + 1])) for i in range(3)],
            [take(build, np.arange(bb[i], bb[i + 1])) for i in range(3)])


def _reference(stream, build, keep, kind, nulls_equal, cond, so, bo):
    """expected output columns: join_maps over the rows the filter keeps, then the condition f >= bid over the pairs"""
    rows = np.flatnonzero(keep)
    st = take(stream, rows)
    if not cond:
        lm, rm = join_maps(build[:1], st[:1], kind, nulls_equal)
    else:
        il, ir = join_maps(build[:1], st[:1], INNER, nulls_equal)
        ok = st[1].values[il] >= build[1].values[ir]
        il, ir = il[ok], ir[ok]
        hit = np.zeros(len(rows), bool)
        hit[il] = True
        if kind == INNER:
            lm, rm = il, ir
        elif kind == SEMI:
            lm, rm = np.flatnonzero(hit), None
        elif kind == ANTI:
            lm, rm = np.flatnonzero(~hit), None
        else:
            lonely = np.flatnonzero(~hit)
            lm, rm = np.r_[il, lonely], np.r_[ir, np.full(len(lonely), INT32_MIN)]
    lm = np.where(lm >= 0, rows[np.maximum(lm, 0)], INT32_MIN)
    want = R.gather([stream[c] for c in so], lm, True)
    if kind not in (SEMI, ANTI):
        want += R.gather([build[c] for c in bo], rm, True)
    return want


def _assert_join(out, want, kind, sid_at, bid_at):
    got = [out.column(c).to_numpy() for c in range(out.num_columns)]
    assert len(got) == len(want) and out.num_rows == len(want[0].values)

    def order(vals, valid):
        s = np.where(valid[sid_at], np.asarray(vals[sid_at], np.int64), -1)
        if kind in (SEMI, ANTI):
            return np.argsort(s, kind="stable")
        return np.lexsort((np.where(valid[bid_at], np.asarray(vals[bid_at], np.int64), -1), s))
    og = order([v for v, _ in got], [ok for _, ok in got])
    ow = order([c.values for c in want], [c.valid for c in want])
    for (v, ok), w in zip(got, want):
        assert np.array_equal(ok[og], w.valid[ow])
        gv = [x for x, k in zip(np.asarray(v, dtype=object)[og], ok[og]) if k]
        wv = [x for x, k in zip(np.asarray(w.values, dtype=object)[ow], w.valid[ow]) if k]
        norm = (lambda x: x if isinstance(x, bytes) else (float(x) if isinstance(x, float) else int(x)))
        if w.typ[0] in (O.FLOAT32, O.FLOAT64):
            assert np.array_equal(np.asarray(gv, np.float64).view(np.int64), np.asarray(wv, np.float64).view(np.int64))
        else:
            assert [norm(x) for x in gv] == [norm(x) for x in wv]


def _run_join(b2, sides, kind, filtered, prune, nulls_equal, cond, target, nparts, ids=(2, 1)):
    """ids: the row-id columns of the stream and the build side, which order both outputs"""
    from spark_rapids_b200 import execs as E
    stream, build, sbatches, bbatches = sides
    gc.collect()
    b2.sync()
    base = b2.device_bytes_in_use()
    src = E.GpuBatchSource([to_table(b2, s) for s in sbatches])
    keep = np.ones(len(stream[0].values), bool)
    if filtered:
        keep = stream[1].values >= 500
        src = E.GpuFilterExec(b2.col(1, b2.INT32, nullable=False) >= b2.lit(500, b2.INT32), src)
    so, bo = ([2, 0, 5, 6, 3], [1, 3, 4, 2]) if prune else (list(range(len(stream))), list(range(len(build))))
    kw = dict(stream_out=so, build_out=bo) if prune else {}
    if cond:
        kw["condition"] = b2.col(1, b2.INT32, nullable=False) >= b2.col(len(stream) + 1, b2.INT32, nullable=False)
    if target is not None:
        kw.update(target_bytes=target, num_sub_partitions=nparts)
    j = E.GpuShuffledHashJoinExec([0], [0], kind, src, E.GpuBatchSource([to_table(b2, b) for b in bbatches]), nulls_equal=nulls_equal, **kw)
    outs = list(j)
    out = b2.concat(outs) if len(outs) > 1 else outs[0]
    want = _reference(stream, build, keep, kind, nulls_equal, cond, so, bo)
    _assert_join(out, want, kind, so.index(ids[0]), len(so) + bo.index(ids[1]) if kind not in (SEMI, ANTI) else None)
    assert j.metrics["numOutputRows"] == out.num_rows and j.metrics["numOutputBatches"] == len(outs)
    stats = j.sub_partition_stats
    del outs, out, j, src
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base
    return stats


def _build_bytes(b2, bbatches):
    return sum(_table_bytes(to_table(b2, b)) for b in bbatches)


@pytest.mark.parametrize("prune", [False, True], ids=["all_columns", "pruned"])
@pytest.mark.parametrize("filtered", [False, True], ids=["no_filter", "filter_below"])
@pytest.mark.parametrize("kind", KINDS)
def test_join_matrix(b2, kind, filtered, prune):
    rng = np.random.default_rng(7 + kind)
    sides = _sides(rng)
    bb = _build_bytes(b2, sides[3])
    for nulls_equal in (False, True):
        for cond in ([False] if kind == FULL_OUTER else [False, True]):
            st = _run_join(b2, sides, kind, filtered, prune, nulls_equal, cond, bb // 5, 16)         # several packed buckets
            assert st["buckets"] == 16 and st["build_bytes"] > 0 and st["stream_bytes"] > 0, st
            assert st["repartitioned"] == 0 or kind == FULL_OUTER, st      # FULL OUTER also splits a bucket whose stream side is over
            st = _run_join(b2, sides, kind, filtered, prune, nulls_equal, cond, int(bb * 0.4), 2)     # each half is over: split again
            assert st["buckets"] == 2 and st["repartitioned"] >= 1, st


@pytest.mark.parametrize("kind", KINDS)
def test_float_keys_join(b2, kind):
    rng = np.random.default_rng(70 + kind)
    sides = _sides(rng, O.FLOAT64)
    bb = _build_bytes(b2, sides[3])
    for nulls_equal in (False, True):
        st = _run_join(b2, sides, kind, False, True, nulls_equal, False, bb // 6, 16)
        assert st["buckets"] == 16, st


# ---- 5. unchanged below the target ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_below_target_is_the_default_join(b2, kind):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(5)
    # the inner + filter shape join_filter_probe_kernel takes: a batch of 2^16 rows or more, stream keys without NULLs
    stream, build, sbatches, bbatches = _sides(rng, sizes=((1 << 16) + 100, 0, 3000), stream_nulls=0)
    bb = _build_bytes(b2, bbatches)
    res = []
    for target in (None, bb, bb * 4):
        src = E.GpuBatchSource([to_table(b2, s) for s in sbatches])
        if kind != FULL_OUTER:
            src = E.GpuFilterExec(b2.col(1, b2.INT32, nullable=False) >= b2.lit(500, b2.INT32), src)
        kw = {} if target is None else dict(target_bytes=target)
        j = E.GpuShuffledHashJoinExec([0], [0], kind, src, E.GpuBatchSource([to_table(b2, b) for b in bbatches]), stream_out=[2, 0], build_out=[1], **kw)
        b2.profile_enable(True)
        try:
            outs = [[c.to_numpy() for c in t.columns()] for t in j]
            names = {k["name"] for k in b2.profile_report()}
        finally:
            b2.profile_enable(False)
        if kind == INNER:
            assert "join_filter_probe_kernel" in names, names
        assert "hash_split_count_kernel" not in names
        assert j.sub_partition_stats == {"buckets": 0, "repartitioned": 0, "build_bytes": 0, "stream_bytes": 0}
        res.append(outs)
    def rows(batch):   # the in-probe filter emits a batch's rows in no fixed order: compare each batch as a multiset of rows
        return sorted(zip(*[[v if k else None for v, k in zip(vals.tolist(), ok)] for vals, ok in batch]), key=repr)
    for other in res[1:]:
        assert len(other) == len(res[0])
        for a, b in zip(res[0], other):
            assert rows(a) == rows(b)


# ---- 6. skew -------------------------------------------------------------------------------------------------------------------
def _int_join(b2, bkeys, skeys, kind, target, nparts=16):
    """INT64 keys with row-id payloads: [key, sid] joined with [key, bid], checked against join_maps"""
    stream = [ocol(skeys, O.INT64), ocol(np.arange(len(skeys), dtype=np.int32), O.INT32)]
    build = [ocol(bkeys, O.INT64), ocol(np.arange(len(bkeys), dtype=np.int32), O.INT32)]
    half = len(bkeys) // 2
    sides = (stream, build, [stream], [take(build, np.arange(half)), take(build, np.arange(half, len(bkeys)))])
    return _run_join(b2, sides, kind, False, False, False, False, target, nparts, ids=(1, 1))


def test_skewed_bucket_is_repartitioned(b2):
    rng = np.random.default_rng(6)
    cand = key_of(rng.permutation(400_000))
    pid = long_pids(cand, 16, 100)
    bkeys = np.r_[cand[pid == 5][:12000], cand[pid != 5][:3000]]          # bucket 5 holds 80 % of the build rows
    skeys = np.r_[rng.choice(bkeys, 20000), cand[-5000:]]
    for kind in KINDS:
        st = _int_join(b2, bkeys, skeys, kind, 64 << 10)
        assert st["buckets"] == 16 and st["repartitioned"] == 1, st


def test_one_key_over_the_target(b2):
    rng = np.random.default_rng(9)
    bkeys = np.r_[np.full(20000, 77, np.int64), key_of(np.arange(3000))]
    skeys = np.r_[np.full(10, 77, np.int64), key_of(rng.integers(0, 6000, 5000))]
    for kind in KINDS:
        st = _int_join(b2, bkeys, skeys, kind, 16 << 10)
        assert st["repartitioned"] >= 1, st


# ---- 7. beyond the allocation limit -------------------------------------------------------------------------------------------
def _host(keys, pays, rows):
    return [[(O.INT64, 0, keys[s:s + rows], None), (O.INT64, 0, pays[s:s + rows], None)] for s in range(0, len(keys), rows)]


def _collect_pairs(node):
    ks, ps = [], []
    for t in node:
        ks.append(t.column(1).to_numpy())
        ps.append(t.column(3).to_numpy())
        del t
    kv, kk = np.concatenate([k[0] for k in ks]), np.concatenate([k[1] for k in ks])
    pv, pk = np.concatenate([p[0] for p in ps]), np.concatenate([p[1] for p in ps])
    return np.where(kk, kv, -1), np.where(pk, pv, -1)


@pytest.mark.parametrize("kind", [INNER, FULL_OUTER])
def test_beyond_the_allocation_limit(b2, limits, kind):
    """INNER: a 96 MiB build side; FULL OUTER: a 96 MiB stream side (8 MiB build side); the limit is 32 MiB above the base"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(17)
    rows = 1 << 17                                           # 2 MiB batches of [INT64 key, INT64 payload]
    nb, ns = (48 * rows, 8 * rows) if kind == INNER else (4 * rows, 48 * rows)
    bk = key_of(rng.permutation(nb))
    sk = np.where(rng.random(ns) < 0.7, bk[rng.integers(0, nb, ns)], key_of(nb + rng.integers(0, nb, ns)))
    bp, sp = np.arange(nb, dtype=np.int64), np.arange(ns, dtype=np.int64) + 10**12
    gc.collect()
    b2.sync()
    base = b2.device_bytes_in_use()
    spilled0 = b2.memory_stats()["spilled_bytes"]
    b2.set_alloc_limit(base + (32 << 20))
    mk = lambda **kw: E.GpuShuffledHashJoinExec([0], [0], kind, E.GpuHostBatchSource(_host(sk, sp, rows)), E.GpuHostBatchSource(_host(bk, bp, rows)), **kw)
    single = mk()
    with pytest.raises(b2.B2Error) as ei:
        single.collect()
    assert ei.value.code == ERR_OOM
    del single, ei
    gc.collect()
    b2.sync()
    node = mk(target_bytes=4 << 20)
    got_s, got_b = _collect_pairs(node)
    assert b2.memory_stats()["spilled_bytes"] > spilled0
    assert node.metrics["numOutputRows"] == len(got_s) and node.sub_partition_stats["buckets"] == 16
    lm, rm = join_maps([ocol(bk, O.INT64)], [ocol(sk, O.INT64)], kind)
    ws = np.where(lm >= 0, sp[np.maximum(lm, 0)], -1)
    wb = np.where(rm >= 0, bp[np.maximum(rm, 0)], -1)
    og, ow = np.lexsort((got_b, got_s)), np.lexsort((wb, ws))
    assert np.array_equal(got_s[og], ws[ow]) and np.array_equal(got_b[og], wb[ow])
    del node
    gc.collect()
    b2.sync()
    assert b2.device_bytes_in_use() == base


# ---- 8. empty edges ------------------------------------------------------------------------------------------------------------
def test_empty_batches_and_exact_target(b2):
    rng = np.random.default_rng(12)
    stream, build, sbatches, bbatches = _sides(rng)
    e_s, e_b = take(stream, np.arange(0)), take(build, np.arange(0))
    sides = (stream, build, [e_s] + sbatches + [e_s], [e_b] + bbatches + [e_b])
    bb = _build_bytes(b2, sides[3])
    for kind in KINDS:
        st = _run_join(b2, sides, kind, False, True, False, False, bb, 16)       # ends exactly at the target: not split
        assert st["buckets"] == 0, st
        st = _run_join(b2, sides, kind, False, True, False, False, bb - 1, 16)
        assert st["buckets"] == 16, st


def test_bucket_with_stream_rows_only(b2):
    """the build keys fill 4 of 16 buckets; the stream's other rows must still come out of LEFT OUTER and ANTI"""
    rng = np.random.default_rng(13)
    cand = key_of(rng.permutation(200_000))
    pid = long_pids(cand, 16, 100)
    bkeys = cand[pid < 4][:6000]
    skeys = np.r_[rng.choice(bkeys, 3000), cand[pid >= 4][:4000]]
    for kind in KINDS:
        st = _int_join(b2, bkeys, skeys, kind, 16 << 10)
        assert st["buckets"] == 16, st
