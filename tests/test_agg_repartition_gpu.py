"""Hash-aggregate repartitioning (GpuMergeAggregateIterator): partial results merged bucket by bucket through spillable hash
buckets, against exact numpy references.  Every repartitioned case also checks that each group key appears in exactly one
output row over all batches, the property bucketing could break."""
import ctypes
import gc

import numpy as np
import pytest

from tests.test_agg_paths_gpu import _words, decimal_result, exact_group_sums, key_of

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_OOM, ERR_SIZE_OVERFLOW = 1, 3, 4
NAN_BITS = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF], dtype=np.uint64)


@pytest.fixture
def limits(b2):
    yield
    b2.set_alloc_limit(0)


# ---- keys: group id -> key values -------------------------------------------------------------------------------------------
# name: (dtype, precision, scale, number of groups, key bytes)
KEY_TYPES = {"bool": ("BOOL8", 0, 0, 2, 1), "int8": ("INT8", 0, 0, 256, 1), "int16": ("INT16", 0, 0, 3000, 2), "int32": ("INT32", 0, 0, 3000, 4),
             "int64": ("INT64", 0, 0, 3000, 8), "float32": ("FLOAT32", 0, 0, 3000, 4), "float64": ("FLOAT64", 0, 0, 3000, 8),
             "date": ("DATE32", 0, 0, 3000, 4), "timestamp": ("TIMESTAMP_US", 0, 0, 3000, 8), "dec32": ("DECIMAL32", 9, 2, 3000, 4),
             "dec64": ("DECIMAL64", 18, 2, 3000, 8), "dec128": ("DECIMAL128", 38, 2, 3000, 16), "string": ("STRING", 0, 0, 3000, 12)}
SHAPES = {name: [name] for name in KEY_TYPES}
SHAPES.update({"two_keys": ["int32", "string"], "four_keys": ["int8", "dec64", "float64", "date"]})


def _key_values(rng, name, ids):
    """values of key type `name` for group ids (distinct ids give distinct keys); for floats, id 0 is NaN in several payloads
    and id 1 is 0.0 or -0.0, chosen per row"""
    n = len(ids)
    if name == "bool":
        return (ids % 2).astype(np.int8)
    if name == "int8":
        return ((ids % 256) - 128).astype(np.int8)
    if name == "int16":
        return (ids * 7 - 20000).astype(np.int16)
    if name in ("int32", "dec32"):
        return (ids * 100_003 - 10**8).astype(np.int32)
    if name == "date":
        return (ids - 1500).astype(np.int32)
    if name in ("int64", "timestamp"):
        return key_of(ids)
    if name == "dec64":
        return ids.astype(np.int64) * 1_000_000_000_007 - 10**17
    if name == "dec128":
        return np.array([(int(i) - 1500) * (10**33 + 7) for i in ids], dtype=object)
    if name == "string":
        return np.array([(b"%x" % i) if i % 3 else (b"long-key-%07d" % i) for i in ids.tolist()], dtype=object)
    ft = np.float32 if name == "float32" else np.float64
    k = (np.where(ids % 2 == 0, 1.0, -1.0) * (ids * 0.37 + 1.0)).astype(ft)
    z = ids == 0
    k[z] = NAN_BITS[rng.integers(0, 4, int(z.sum()))].view(np.float64).astype(ft)
    o = ids == 1
    k[o] = np.array([0.0, -0.0], dtype=ft)[rng.integers(0, 2, int(o.sum()))]
    return k


def _norm(v):
    """an output key value, comparable with the reference: NaN -> 'nan', -0.0 -> 0.0, NULL -> None"""
    if isinstance(v, float):
        return "nan" if v != v else (0.0 if v == 0 else v)
    return v.decode() if isinstance(v, bytes) else v


def _to_column(b2, name, vals, valid):
    dt, _, scale, _, _ = KEY_TYPES[name]
    v = None if valid is None or valid.all() else valid
    if dt == "STRING":
        offs = np.zeros(len(vals) + 1, np.int32)
        offs[1:] = np.cumsum([len(s) for s in vals])
        chars = np.frombuffer(b"".join(vals), dtype=np.uint8) if len(vals) else np.zeros(0, np.uint8)
        return b2.Column.from_string_buffers(chars, offs, valid=v)
    return b2.Column.from_numpy(vals, dtype=getattr(b2, dt), scale=scale, valid=v)


def _key_expr(b2, name, i, nullable):
    dt, p, s, _, _ = KEY_TYPES[name]
    return b2.col(i, getattr(b2, dt), p, s, nullable=nullable)


class Data:
    """rows of a key shape with an INT64 value column (10 % NULL): group ids, key columns per batch and the exact reference
    {normalised key tuple: (SUM, COUNT, COUNT_ALL, MIN, MAX)}"""

    def __init__(self, b2, shape, nrows=40_000, nbatches=8, seed=0, nullable=False):
        """nullable: the first key column is nullable, and one extra group has the NULL key"""
        rng = np.random.default_rng(seed)
        names = SHAPES[shape]
        base = min(KEY_TYPES[n][3] for n in names)
        ngroups = base + nullable
        null_group = base if nullable else None
        g = rng.integers(0, ngroups, nrows)
        g[:ngroups] = np.arange(ngroups)
        rng.shuffle(g)
        v = rng.integers(-10**6, 10**6, nrows)
        vok = rng.random(nrows) >= 0.1
        self.names, self.nk = names, len(names)
        kcols = [_key_values(rng, n, g) for n in names]
        kvalid = [None if (null_group is None or j) else g != null_group for j in range(len(names))]
        self.nullable = nullable
        bounds = np.linspace(0, nrows, nbatches + 1).astype(int)
        self.batches = []
        for s, e in zip(bounds[:-1], bounds[1:]):
            cols = [_to_column(b2, n, k[s:e], None if kv is None else kv[s:e]) for n, k, kv in zip(names, kcols, kvalid)]
            cols.append(b2.Column.from_numpy(v[s:e], valid=vok[s:e]))
            self.batches.append(b2.Table.from_columns(cols))
        ids = np.arange(ngroups)
        want_keys = [[_norm(x) for x in (_key_values(np.random.default_rng(0), n, ids).tolist())] for n in names]
        for j in range(len(names)):
            for i in range(ngroups):
                if names[j] in ("float32", "float64") and i == 0:
                    want_keys[j][i] = "nan"
                if names[j] in ("float32", "float64") and i == 1:
                    want_keys[j][i] = 0.0
                if isinstance(want_keys[j][i], float) and names[j] == "float32":
                    want_keys[j][i] = float(np.float32(want_keys[j][i]))
                if names[j] == "bool":
                    want_keys[j][i] = bool(want_keys[j][i])
                if kvalid[j] is not None and i == null_group:
                    want_keys[j][i] = None
        self.want = {}
        for i in range(ngroups):
            m = g == i
            vv = v[m & vok]
            agg = (int(vv.sum()) if len(vv) else None, len(vv), int(m.sum()), int(vv.min()) if len(vv) else None, int(vv.max()) if len(vv) else None)
            self.want[tuple(want_keys[j][i] for j in range(len(names)))] = agg
        self.bytes = ngroups * (sum(KEY_TYPES[n][4] for n in names) + 40)   # about the partials of one batch

    def pre(self, b2):
        return [_key_expr(b2, n, j, self.nullable and j == 0) for j, n in enumerate(self.names)] + [b2.col(self.nk, b2.INT64, nullable=True)]

    def specs(self, b2):
        c = self.nk
        return [(b2.AGG_SUM, c, b2.INT64, 0, 0), (b2.AGG_COUNT, c), (b2.AGG_COUNT_ALL, 0), (b2.AGG_MIN, c, 0, 0, 0), (b2.AGG_MAX, c, 0, 0, 0)]


def _rows(batches, nk):
    """output batches -> list of (normalised key tuple, aggregate tuple)"""
    out = []
    for t in batches:
        cols = t.to_pylists()
        for r in zip(*cols):
            out.append((tuple(_norm(x) for x in r[:nk]), tuple(r[nk:])))
    return out


def _check(rows, want):
    keys = [k for k, _ in rows]
    assert len(set(keys)) == len(keys), "a group key appears in more than one output row"
    assert dict(rows) == want


def _plan(b2, d, plan, target, k):
    from spark_rapids_b200 import execs as E
    kw = {} if target is None else dict(target_bytes=target, num_buckets=k)
    src = E.GpuBatchSource(d.batches)
    keys = list(range(d.nk))
    if plan == "complete":
        return E.GpuHashAggregateExec(src, keys, d.specs(b2), pre_project=d.pre(b2), mode="complete", **kw), None
    partial = E.GpuHashAggregateExec(src, keys, d.specs(b2), pre_project=d.pre(b2), **kw)
    return E.GpuHashAggregateExec(partial, keys, d.specs(b2), mode="final", **kw), partial


def _run(b2, node):
    outs = list(node)
    assert node.metrics["numOutputBatches"] == len(outs)
    assert node.metrics["numOutputRows"] == sum(t.num_rows for t in outs)
    return outs


# ---- 2. forced repartition: every key type, K = 2, 16, 256 --------------------------------------------------------------------
@pytest.mark.parametrize("plan", ["complete", "partial_final"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_forced_repartition(b2, shape, plan):
    d = Data(b2, shape, seed=len(shape), nullable=shape not in ("two_keys", "four_keys"))
    target = max(16, d.bytes // 6)
    for k in (2, 16, 256):
        node, partial = _plan(b2, d, plan, target, k)
        outs = _run(b2, node)
        _check(_rows(outs, d.nk), d.want)
        st = node.repartition_stats
        assert st["buckets"] == k and st["bytes_split"] > 0, st
        if partial is not None:
            assert partial.repartition_stats["buckets"] == k
        if k == 2:
            assert st["resplit"] >= 1 and st["depth"] >= 1, st


# ---- 1. below the target: the default path --------------------------------------------------------------------------------
def _bits(t):
    """a batch as a sorted list of rows of raw values (floats by their bits, except that which NaN payload or sign of zero
    stands for its group depends on which row reached the hash table first): the hash tables place groups by atomics, so
    row order inside a batch is not compared"""
    cols = []
    for c in t.columns():
        vals, ok = c.to_numpy()
        if vals.dtype.kind == "f":
            vals = np.where(np.isnan(vals), np.nan, np.where(vals == 0, 0.0, vals)).astype(vals.dtype)
            vals = vals.view("u%d" % vals.dtype.itemsize)
        cols.append([v if o else None for v, o in zip(vals.tolist(), ok)])
    return sorted(zip(*cols), key=repr)


@pytest.mark.parametrize("mode", ["partial", "complete", "final"])
def test_below_target_is_the_default_path(b2, mode):
    from spark_rapids_b200 import execs as E
    d = Data(b2, "four_keys", seed=11)
    specs = d.specs(b2)
    res = []
    for target in (None, 1 << 40):
        kw = {} if target is None else dict(target_bytes=target)
        if mode == "final":   # several batches of aggregation buffers, keys repeating between them
            src = E.GpuBatchSource([b2.groupby(t, list(range(d.nk)), specs) for t in d.batches])
            node = E.GpuHashAggregateExec(src, list(range(d.nk)), specs, mode="final", **kw)
        else:
            node = E.GpuHashAggregateExec(E.GpuBatchSource(d.batches), list(range(d.nk)), specs, pre_project=d.pre(b2), mode=mode, **kw)
        b2.profile_enable(True)
        try:
            outs = _run(b2, node)
            names = sorted(k["name"] for k in b2.profile_report())
        finally:
            b2.profile_enable(False)
        assert "hash_split_count_kernel" not in names
        assert node.repartition_stats == {"buckets": 0, "resplit": 0, "bytes_split": 0, "depth": 0}
        res.append(([_bits(t) for t in outs], names))
        if mode != "partial":
            _check(_rows(outs, d.nk), d.want)
    assert res[0] == res[1]


# ---- 3. second level and the depth bound ---------------------------------------------------------------------------------------
def test_bucket_over_the_target_is_split_again(b2):
    d = Data(b2, "int64", nrows=200_000, seed=3)
    node, _ = _plan(b2, d, "complete", d.bytes // 40, 16)
    _check(_rows(_run(b2, node), 1), d.want)
    st = node.repartition_stats
    assert st["buckets"] == 16 and st["resplit"] >= 1 and st["depth"] >= 1, st


def test_one_key_reaches_the_depth_bound(b2):
    """300 FINAL input batches that all carry key 7 (three rows each): every level leaves one non-empty bucket over the target,
    so the bucket is split ten times and then merged as it is"""
    from spark_rapids_b200 import execs as E
    specs = [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]
    batches = [b2.Table.from_columns([b2.Column.from_numpy(np.full(3, 7, np.int64)), b2.Column.from_numpy(np.array([i, 1, -1], np.int64)),
                                      b2.Column.from_numpy(np.full(3, 2, np.int64))]) for i in range(300)]
    node = E.GpuHashAggregateExec(E.GpuBatchSource(batches), [0], specs, mode="final", target_bytes=16, num_buckets=16)
    outs = _run(b2, node)
    assert [r for t in outs for r in t.to_rows()] == [(7, sum(range(300)), 1800)]
    st = node.repartition_stats
    assert st["buckets"] == 16 and st["resplit"] == 10 and st["depth"] == 10, st


# ---- 4. merge neighbours ----------------------------------------------------------------------------------------------------
def test_merge_neighbours_never_buckets(b2):
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(4)
    keys = key_of(np.arange(1000))
    vals = [rng.integers(-10**9, 10**9, 1000) for _ in range(200)]
    batches = [b2.Table.from_columns([b2.Column.from_numpy(rng.permutation(keys)), b2.Column.from_numpy(v)]) for v in vals]
    one = 1000 * 24                                                      # one partial: INT64 key, SUM, COUNT_ALL
    pre = [b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.INT64, nullable=False)]
    specs = [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]
    # the batches carry the keys in different orders: the value of key i in batch b is found through the permutation
    tot = {}
    for t, v in zip(batches, vals):
        k = t.column(0).to_numpy()[0]
        for kk, vv in zip(k.tolist(), v.tolist()):
            tot[kk] = tot.get(kk, 0) + vv
    node = E.GpuHashAggregateExec(E.GpuBatchSource(batches), [0], specs, pre_project=pre, mode="complete", target_bytes=5 * one)
    outs = _run(b2, node)
    rows = [r for t in outs for r in t.to_rows()]
    assert len(outs) == 1 and sorted(rows) == sorted((k, s, 200) for k, s in tot.items())
    assert node.repartition_stats["buckets"] == 0


# ---- 5. decimal SUM overflow through the buckets --------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", ["complete_not_null", "complete_nullable", "partial_final"])
def test_decimal_overflow_survives_buckets(b2, plan):
    """group 0 overflows 10^38 inside batch 0 (and in total); with nullable input group 1 is all NULL; both stay NULL, every
    other group's sum is exact"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(5)
    n, ngroups, nb = 40_000, 3000, 8
    g = rng.integers(2, ngroups, n)
    lo, hi = _words([int(x) for x in rng.integers(-10**15, 10**15, n)])
    over_lo, over_hi = _words([4 * 10**37] * 3)
    g = np.r_[np.zeros(3, np.int64), g]
    lo, hi = np.r_[over_lo, lo], np.r_[over_hi, hi]                       # batch 0 starts with the overflowing rows
    valid = np.ones(len(g), bool)
    nullable = plan != "complete_not_null"
    if nullable:
        valid[3:] = rng.random(n) >= 0.1
        valid[g == 1] = False
    keys, tot, cnt = exact_group_sums(g, lo, hi, valid)
    want = dict(zip(key_of(keys).tolist(), decimal_result(tot, cnt, 38)))
    assert want[int(key_of(np.array([0]))[0])] is None
    bounds = np.linspace(0, len(g), nb + 1).astype(int)
    batches = []
    for s, e in zip(bounds[:-1], bounds[1:]):
        dec = np.stack([lo[s:e].view(np.uint64), hi[s:e].view(np.uint64)], axis=1)
        batches.append(b2.Table.from_columns([b2.Column.from_numpy(key_of(g[s:e])),
                                              b2.Column.from_numpy(dec, dtype=b2.DECIMAL128, valid=None if valid[s:e].all() else valid[s:e])]))
    pre = [b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.DECIMAL128, 38, 0, nullable=nullable)]
    specs = [(b2.AGG_SUM, 1, b2.DECIMAL128, 0, 38)]
    target = ngroups * 40 // 6
    src = E.GpuBatchSource(batches)
    if plan == "partial_final":
        partial = E.GpuHashAggregateExec(src, [0], specs, pre_project=pre, target_bytes=target)
        node = E.GpuHashAggregateExec(partial, [0], specs, mode="final", target_bytes=target)
    else:
        node = E.GpuHashAggregateExec(src, [0], specs, pre_project=pre, mode="complete", target_bytes=target)
    outs = _run(b2, node)
    assert all(t.num_columns == 2 for t in outs)
    rows = [r for t in outs for r in t.to_rows()]
    assert len({k for k, _ in rows}) == len(rows)
    assert dict(rows) == want
    assert node.repartition_stats["buckets"] == 16


# ---- 6. partials larger than the allocation limit ------------------------------------------------------------------------------
def test_partials_beyond_the_allocation_limit(b2, limits):
    """32 batches of 2^17 rows, about 3 M groups: 96 MiB of partials against a limit 32 MiB above the base"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(6)
    rows, nb = 1 << 17, 32
    g = rng.integers(0, 3_000_000, rows * nb)
    keys, vals = key_of(g), rng.integers(-10**9, 10**9, rows * nb)
    host = [[(b2.INT64, 0, keys[s:s + rows], None), (b2.INT64, 0, vals[s:s + rows], None)] for s in range(0, rows * nb, rows)]
    pre = [b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.INT64, nullable=False)]
    specs = [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]
    mk = lambda **kw: E.GpuHashAggregateExec(E.GpuHostBatchSource(host), [0], specs, pre_project=pre, mode="complete", **kw)
    gc.collect()
    b2.sync()
    base = b2.device_bytes_in_use()
    spilled0 = b2.memory_stats()["spilled_bytes"]
    b2.set_alloc_limit(base + (32 << 20))
    single = mk()
    with pytest.raises(b2.B2Error) as ei:
        single.collect()
    assert ei.value.code == ERR_OOM
    del single, ei
    gc.collect()
    b2.sync()
    node = mk(target_bytes=1 << 20)   # a merge's workspace must fit beside the pieces that cannot leave the device
    got_k, got_s, got_c = [], [], []
    for t in node:
        got_k.append(t.column(0).to_numpy()[0])
        got_s.append(t.column(1).to_numpy()[0])
        got_c.append(t.column(2).to_numpy()[0])
        del t
    assert b2.memory_stats()["spilled_bytes"] > spilled0
    assert node.repartition_stats["buckets"] == 16
    k, s, c = np.concatenate(got_k), np.concatenate(got_s), np.concatenate(got_c)
    order = np.argsort(g, kind="stable")
    sg = g[order]
    starts = np.flatnonzero(np.r_[True, sg[1:] != sg[:-1]])
    wk, ws, wc = key_of(sg[starts]), np.add.reduceat(vals[order], starts), np.diff(np.r_[starts, len(g)])
    o, wo = np.argsort(k), np.argsort(wk)
    assert np.array_equal(k[o], wk[wo]) and np.array_equal(s[o], ws[wo]) and np.array_equal(c[o], wc[wo])
    del node
    gc.collect()
    b2.sync()
    b2.set_alloc_limit(0)
    assert b2.device_bytes_in_use() == base


# ---- 7. more than 2^31 - 1 groups -------------------------------------------------------------------------------------------
def test_more_groups_than_one_batch_can_hold(b2):
    """2^31 + 2^20 distinct INT32 keys (all 2^32 bit patterns are distinct values) and 2^20 of them once more, COUNT_ALL: the
    single merge passes 2^31 - 1 rows; the buckets give batches below 2^31 rows whose totals are checked on the device"""
    from spark_rapids_b200 import execs as E
    distinct, again, step = (1 << 31) + (1 << 20), 1 << 20, 1 << 27
    pre = [b2.col(0, b2.INT32, nullable=False)]
    specs = [(b2.AGG_COUNT_ALL, 0)]

    def source():
        ts = [b2.Table.from_columns([b2.Column.from_numpy(np.arange(s, min(s + step, distinct), dtype=np.int64).astype(np.int32))])
              for s in range(0, distinct, step)]
        ts.append(b2.Table.from_columns([b2.Column.from_numpy(np.arange(again, dtype=np.int32))]))
        return E.GpuBatchSource(ts)

    single = E.GpuHashAggregateExec(source(), [0], specs, pre_project=pre, mode="complete")
    with pytest.raises(b2.B2Error) as ei:
        single.collect()
    assert ei.value.code == ERR_SIZE_OVERFLOW
    del single, ei
    gc.collect()
    node = E.GpuHashAggregateExec(source(), [0], specs, pre_project=pre, mode="complete", target_bytes=4 << 30)
    groups = total = batches = 0
    lo, hi = 2, 0
    for t in node:
        assert t.num_rows < 1 << 31
        s, mn, mx = b2.reduce(t, [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_MIN, 1, 0, 0, 0), (b2.AGG_MAX, 1, 0, 0, 0)]).to_rows()[0]
        groups += t.num_rows
        total += s
        lo, hi = min(lo, mn), max(hi, mx)
        batches += 1
        del t
    assert groups == distinct and total == distinct + again and (lo, hi) == (1, 2)
    assert batches >= 2 and node.metrics["numOutputBatches"] == batches and node.repartition_stats["buckets"] == 16


# ---- 8. errors and interfaces --------------------------------------------------------------------------------------------------
def test_invalid_arguments_and_keyless(b2):
    from spark_rapids_b200 import execs as E
    from spark_rapids_b200._lib import lib
    d = Data(b2, "int64", nrows=5000, nbatches=3)
    for target, k in ((0, 16), (-1, 16), (1 << 20, 1), (1 << 20, 257)):
        with pytest.raises(b2.B2Error) as ei:
            _plan(b2, d, "complete", target, k)
        assert ei.value.code == ERR_INVALID
    src = E.GpuBatchSource(d.batches)
    for rc in (lib.b2_exec_aggregate_set_repartitioning(src.h, 1 << 20, 16), lib.b2_exec_aggregate_repartition_stats(src.h, (ctypes.c_int64 * 4)())):
        assert rc == ERR_INVALID
    node, _ = _plan(b2, d, "complete", 1 << 10, 16)
    node.next()
    assert lib.b2_exec_aggregate_set_repartitioning(node.h, 1 << 20, 16) == ERR_INVALID     # already running
    # keyless: accepted, no effect
    specs = [(b2.AGG_SUM, 0, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]
    res = []
    for kw in ({}, dict(target_bytes=16, num_buckets=2)):
        node = E.GpuHashAggregateExec(E.GpuBatchSource(d.batches), [], specs, pre_project=[b2.col(1, b2.INT64, nullable=True)], mode="complete", **kw)
        res.append(_run(b2, node)[0].to_rows())
        assert node.repartition_stats["buckets"] == 0
    assert res[0] == res[1]
