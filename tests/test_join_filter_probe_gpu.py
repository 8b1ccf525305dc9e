"""The filter evaluated inside the FK -> PK join probe (join_filter_probe_kernel, b2_join_probe_filter): the same pairs, match
count and passing-row count as the selection-vector path (b2_filter_row_ids + b2_join_probe_sel) and as numpy, and the
kernel that ran, read from the kernel timings."""
import operator

import numpy as np
import pytest

from oracle import spark_cpu as O
from tests.test_join_paths_gpu import join_maps

pytestmark = pytest.mark.gpu

FUSED, SEL_FILTER, SEL_PROBE = "join_filter_probe_kernel", "simple_filter_ids_kernel", "join_probe_distinct1_kernel"
TILE = 8192                      # rows per tile of the fused kernel
OPS = [operator.eq, operator.ne, operator.lt, operator.le, operator.gt, operator.ge]


def passing_pairs(skey, svalid, keep, bkey, bvalid):
    """sorted (stream row, build row) pairs of the passing stream rows, from the exact reference (test_join_paths_gpu)"""
    rows = np.flatnonzero(keep)
    lm, rm = join_maps([O.OCol(bkey, bvalid, (O.INT64, 0, 0))], [O.OCol(skey[rows], svalid[rows], (O.INT64, 0, 0))], 0)
    return sorted(zip(rows[lm].tolist(), rm.tolist()))


def pairs_of(lm, rm):
    return sorted(zip(lm.to_numpy()[0].astype(np.int64).tolist(), rm.to_numpy()[0].astype(np.int64).tolist()))


def check(b2, stream_cols, key_col, pred, keep, bkey, bvalid=None, skey_valid=None, fused=True):
    """probe through b2_join_probe_filter and through the selection-vector path; compare both with numpy"""
    skey = stream_cols[key_col]
    n = len(skey)
    bvalid = np.ones(len(bkey), bool) if bvalid is None else bvalid
    svalid = np.ones(n, bool) if skey_valid is None else skey_valid
    table = b2.Table.from_columns([b2.Column.from_numpy(c, valid=(svalid if (i == key_col and skey_valid is not None) else None))
                                   for i, c in enumerate(stream_cols)])
    ht = b2.JoinHashTable(b2.Table.from_columns([b2.Column.from_numpy(bkey, valid=None if bvalid.all() else bvalid)]))
    prog = b2.Program([pred])
    b2.profile_enable(True)
    lm, rm, npass = ht.probe_filter(table, key_col, prog)
    names = {k["name"] for k in b2.profile_report()}
    b2.profile_enable(False)
    assert (FUSED in names) == fused, names
    if fused:
        assert SEL_FILTER not in names and SEL_PROBE not in names, names
    want = passing_pairs(skey.astype(np.int64), svalid, keep, bkey.astype(np.int64), bvalid)
    got = pairs_of(lm, rm)
    assert npass == int(keep.sum())
    assert len(lm) == len(want)
    assert got == want
    sel = b2.filter_row_ids(prog, table)
    assert len(sel) == npass
    keys = b2.Table.from_columns([b2.Column.from_numpy(skey, valid=None if skey_valid is None else svalid)])
    slm, srm = ht.probe(keys, b2.JOIN_INNER, selection=sel)
    assert pairs_of(slm, srm) == got
    return got


def dtype_of(b2, npt):
    return {np.int8: b2.INT8, np.int16: b2.INT16, np.int32: b2.INT32, np.int64: b2.INT64}[npt]


@pytest.mark.parametrize("kt", [np.int32, np.int64])
@pytest.mark.parametrize("nb", [100_000, 600_000])          # below 2^18 build rows: no Bloom filter; above: Bloom filter on
def test_keys_and_build_sizes(b2, kt, nb):
    rng = np.random.default_rng(1)
    info = np.iinfo(kt)
    n = 9 * TILE + 123                                       # not a multiple of the tile
    pool = np.concatenate([np.array([info.min, info.min + 1, -1, 0, 1, info.max - 1, info.max], kt),
                           rng.integers(info.min, info.max, 2 * nb, dtype=kt)])
    pool = np.unique(pool)
    bkey = rng.permutation(pool)[:nb]
    bkey = np.unique(np.concatenate([bkey, np.array([info.min, -1, 0, info.max], kt)]))
    skey = np.where(rng.random(n) < 0.5, rng.choice(bkey, n), rng.integers(info.min, info.max, n, dtype=kt)).astype(kt)
    skey[:4] = [info.min, -1, 0, info.max]
    d = rng.integers(0, 1000, n).astype(np.int32)
    keep = d >= 500
    keep[:4] = True
    d[:4] = 999
    pred = b2.col(1, b2.INT32, nullable=False) >= b2.lit(500, b2.INT32)
    check(b2, [skey, d], 0, pred, keep, bkey)


@pytest.mark.parametrize("width", [1, 2, 4, 8])
def test_term_widths_ops_and_limits(b2, width):
    """every comparison on a column of each width, with literals at the type's limits and inside its range"""
    npt = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[width]
    info = np.iinfo(npt)
    rng = np.random.default_rng(10 + width)
    n = 8 * TILE + 77
    nb = 50_000
    bkey = rng.permutation(200_000)[:nb].astype(np.int64)
    skey = rng.integers(0, 200_000, n).astype(np.int64)
    v = rng.integers(info.min, info.max, n, dtype=npt, endpoint=True)
    v[:6] = [info.min, info.min, info.max, info.max, 0, -1]
    dt = dtype_of(b2, npt)
    for lit in (info.min, info.max, 0, int(v[100])):
        for op in OPS:
            pred = op(b2.col(1, dt, nullable=False), b2.lit(int(lit), dt))
            check(b2, [skey, v], 0, pred, op(v, npt(lit)), bkey)


@pytest.mark.parametrize("nterms", [1, 2, 3, 5, 8])
def test_conjunctions(b2, nterms):
    """1 to 8 terms over columns of mixed widths, each with its own operator"""
    rng = np.random.default_rng(100 + nterms)
    n = 9 * TILE + 5
    bkey = rng.permutation(1 << 20)[:300_000].astype(np.int64)
    skey = rng.integers(0, 1 << 20, n).astype(np.int64)
    types = [np.int8, np.int16, np.int32, np.int64]
    cols, keep, pred = [skey], np.ones(n, bool), None
    for k in range(nterms):
        npt = types[k % 4]
        info = np.iinfo(npt)
        c = rng.integers(-50, 50, n).astype(npt)
        op = OPS[(k * 5 + nterms) % 6]
        lit = int(rng.integers(-20, 20)) if op not in (operator.eq, operator.ne) else int(rng.integers(-3, 3))
        if k == 7:
            op, lit = operator.ge, int(info.min)             # a term every row passes
        cols.append(c)
        keep &= op(c, npt(lit))
        term = op(b2.col(k + 1, dtype_of(b2, npt), nullable=False), b2.lit(lit, dtype_of(b2, npt)))
        pred = term if pred is None else pred & term
    check(b2, cols, 0, pred, keep, bkey)


@pytest.mark.parametrize("case", ["none", "all", "half", "sparse", "last_row_of_tile"])
def test_selectivity(b2, case):
    rng = np.random.default_rng(7)
    n = 10 * TILE + 4000
    bkey = np.arange(0, 2_000_000, 3, dtype=np.int64)             # 667k rows: Bloom filter on
    skey = rng.integers(0, 2_000_000, n).astype(np.int64)
    d = rng.integers(0, 100_000, n).astype(np.int32)
    if case == "last_row_of_tile":
        d[:] = 0
        d[2 * TILE - 1] = 5                                        # only the last row of the second tile passes
        skey[2 * TILE - 1] = 3 * 1234
    thr = {"none": 100_000, "all": -1, "half": 50_000, "sparse": 99_500, "last_row_of_tile": 0}[case]
    pred = b2.col(1, b2.INT32, nullable=False) > b2.lit(thr, b2.INT32)
    got = check(b2, [skey, d], 0, pred, d > thr, bkey)
    if case == "last_row_of_tile":
        assert got == [(2 * TILE - 1, 1234)]


@pytest.mark.parametrize("n,fused", [((1 << 16) - 1, False), (1 << 16, True), ((1 << 16) + 1, True)])
def test_row_threshold(b2, n, fused):
    rng = np.random.default_rng(3)
    bkey = rng.permutation(400_000)[:300_000].astype(np.int32)
    skey = rng.integers(0, 400_000, n).astype(np.int32)
    d = rng.integers(0, 10, n).astype(np.int16)
    pred = b2.col(1, b2.INT16, nullable=False) != b2.lit(4, b2.INT16)
    check(b2, [skey, d], 0, pred, d != 4, bkey, fused=fused)


def test_duplicate_build_keys_fall_back(b2):
    rng = np.random.default_rng(4)
    n = 9 * TILE + 9
    bkey = rng.integers(0, 50_000, 100_000).astype(np.int64)      # many duplicates: not a distinct build side
    skey = rng.integers(0, 60_000, n).astype(np.int64)
    d = rng.integers(0, 100, n).astype(np.int32)
    pred = b2.col(1, b2.INT32, nullable=False) < b2.lit(30, b2.INT32)
    check(b2, [skey, d], 0, pred, d < 30, bkey, fused=False)


def test_nullable_key_falls_back(b2):
    rng = np.random.default_rng(5)
    n = 9 * TILE + 9
    bkey = rng.permutation(100_000)[:60_000].astype(np.int64)
    skey = rng.integers(0, 100_000, n).astype(np.int64)
    valid = rng.random(n) > 0.1
    d = rng.integers(0, 100, n).astype(np.int32)
    pred = b2.col(1, b2.INT32, nullable=False) < b2.lit(70, b2.INT32)
    check(b2, [skey, d], 0, pred, d < 70, bkey, skey_valid=valid, fused=False)


def test_odd_offset_slice(b2):
    """a slice at an odd offset (what split-and-retry makes): slices are copies into fresh 16-byte aligned buffers, so the
    fused kernel takes them like any batch"""
    rng = np.random.default_rng(6)
    n = 9 * TILE
    bkey = rng.permutation(100_000)[:60_000].astype(np.int64)
    skey = rng.integers(0, 100_000, n + 1).astype(np.int64)
    d = rng.integers(0, 100, n + 1).astype(np.int32)
    full = b2.Table.from_columns([b2.Column.from_numpy(skey), b2.Column.from_numpy(d)])
    part = b2.slice_table(full, 1, n + 1)
    ht = b2.JoinHashTable(b2.Table.from_columns([b2.Column.from_numpy(bkey)]))
    prog = b2.Program([b2.col(1, b2.INT32, nullable=False) >= b2.lit(40, b2.INT32)])
    b2.profile_enable(True)
    lm, rm, npass = ht.probe_filter(part, 0, prog)
    names = {k["name"] for k in b2.profile_report()}
    b2.profile_enable(False)
    assert FUSED in names, names
    keep = d[1:] >= 40
    assert npass == int(keep.sum())
    assert pairs_of(lm, rm) == passing_pairs(skey[1:], np.ones(n, bool), keep, bkey, np.ones(len(bkey), bool))


def test_exec_path_several_batches(b2):
    """GpuFilterExec under GpuShuffledHashJoinExec: every batch goes through the fused kernel; numOutputRows is the sum of
    the passing rows"""
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(8)
    nbatch, per = 3, 9 * TILE + 17
    ns = nbatch * per
    skey = rng.integers(0, 1_000_000, ns).astype(np.int64)
    sdate = rng.integers(8000, 11000, ns).astype(np.int32)
    sval = rng.integers(0, 1 << 40, ns).astype(np.int64)
    bkey = rng.permutation(1_000_000)[:400_000].astype(np.int64)
    bval = bkey * 3 + 1
    batches = [b2.Table.from_columns([b2.Column.from_numpy(skey[i * per:(i + 1) * per]), b2.Column.from_numpy(sdate[i * per:(i + 1) * per], dtype=b2.DATE32),
                                      b2.Column.from_numpy(sval[i * per:(i + 1) * per])]) for i in range(nbatch)]
    bt = b2.Table.from_columns([b2.Column.from_numpy(bkey), b2.Column.from_numpy(bval)])
    flt = E.GpuFilterExec(b2.Program([b2.col(1, b2.DATE32, nullable=False) > b2.lit(9204, b2.DATE32)]), E.GpuBatchSource(batches))
    j = E.GpuShuffledHashJoinExec([0], [0], b2.JOIN_INNER, flt, E.GpuBatchSource([bt]), stream_out=[0, 2], build_out=[1])
    b2.profile_enable(True)
    out = j.collect()
    prof = {k["name"]: k["launches"] for k in b2.profile_report()}
    b2.profile_enable(False)
    assert prof.get(FUSED) == nbatch and SEL_FILTER not in prof and SEL_PROBE not in prof, prof
    keep = sdate > 9204
    lut = np.full(1_000_000, -1, dtype=np.int64)
    lut[bkey] = bval
    hit = keep & (lut[skey] >= 0)
    assert sorted(out.to_rows()) == sorted(zip(skey[hit].tolist(), sval[hit].tolist(), lut[skey[hit]].tolist()))
    assert flt.metrics["numOutputRows"] == int(keep.sum())
