"""The radix group-by's fused materialise + first pass (radix_rows_scatter_kernel after a count pass over the key columns)
against the separate path it replaces (radix_rows_kernel, then every scatter pass), which B2_AGG_NO_FUSED_FIRST_PASS forces.
Every case runs both ways, asserts from the kernel timings which path ran, and compares both with exact integer references:
 * one- and two-word keys; INT64 SUM + COUNT, q3's DECIMAL128 SUM of price * (1 - disc) (the specialised aggregation
   kernel) and MIN / MAX (the generic one);
 * row counts that are multiples of neither the fused tile (2048 rows) nor the scatter's or the VM's tiles;
 * the fewest partitions the radix regime reaches (it starts above 2^20 rows: 10 hash bits, one pass after the fused one)
   and a case that needs 17 bits, so two passes follow the fused one;
 * a fused predicate, which keeps the separate path (its rows are compacted);
 * q3's regime, millions of groups from about 2.5 times as many rows, run twice with identical results.
Keys are k = (i * A) mod G for row i: every group is present, and its rows are known in closed form where a sort of the
reference would be slow."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SWITCH = "B2_AGG_NO_FUSED_FIRST_PASS"
FUSED = {"radix_rows_scatter_kernel", "part_tile_hist_kernel(keys)"}
A = 1_000_003


def _run(b2, fn, fused):
    """fn() with kernel timing on, through the fused first pass or the separate one -> (result, {kernel name: launches})"""
    if fused:
        os.environ.pop(SWITCH, None)
    else:
        os.environ[SWITCH] = "1"
    b2.profile_enable(True)
    try:
        r = fn()
        ran = {k["name"]: k["launches"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
        os.environ.pop(SWITCH, None)
    return r, ran


def _assert_path(ran, fused, scatter_passes):
    if fused:
        assert FUSED <= set(ran) and "radix_rows_kernel" not in ran, ran
        assert ran.get("part_scatter2_kernel", 0) == scatter_passes - 1, ran
    else:
        assert "radix_rows_kernel" in ran and not FUSED & set(ran), ran
        assert ran.get("part_scatter2_kernel", 0) == scatter_passes, ran


def _keys(n, g):
    return (np.arange(n, dtype=np.int64) * A) % g


def _by_key(out, nk):
    """output columns as numpy arrays, rows ordered by the first key column"""
    cols = [out.column(c).to_numpy()[0] for c in range(out.num_columns)]
    o = np.argsort(cols[0], kind="stable")
    return [c[o] for c in cols]


def _reference(k0, v):
    """per key (ascending): present keys, exact int64 sums, counts, minima, maxima of v"""
    order = np.argsort(k0, kind="stable")
    sk, sv = k0[order], v[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    return (sk[starts], np.add.reduceat(sv, starts), np.diff(np.r_[starts, len(sk)]), np.minimum.reduceat(sv, starts),
            np.maximum.reduceat(sv, starts))


def _q3_like(b2, n, g, nk, seed):
    """(table, program, spec, reference) for SUM(price * (1 - disc)) over nk key columns (INT64 [, DATE32, INT32])"""
    rng = np.random.default_rng(seed)
    k0 = _keys(n, g)
    price = rng.integers(90_000, 10_494_951, n, dtype=np.int64)
    disc = rng.integers(0, 11, n, dtype=np.int64)
    cols = [b2.Column.from_numpy(k0)]
    exprs = [b2.col(0, b2.INT64, nullable=False)]
    if nk >= 2:
        cols.append(b2.Column.from_numpy((8000 + k0 % 2557).astype(np.int32), dtype=b2.DATE32))
        exprs.append(b2.col(1, b2.DATE32, nullable=False))
    if nk >= 3:
        cols.append(b2.Column.from_numpy((k0 % 5).astype(np.int32)))
        exprs.append(b2.col(2, b2.INT32, nullable=False))
    nkc = len(cols)
    cols += [b2.Column.from_numpy(price, dtype=b2.DECIMAL64, scale=2), b2.Column.from_numpy(disc, dtype=b2.DECIMAL64, scale=2)]
    one = b2.lit(1, b2.DECIMAL32, 1, 0)
    pr, di = b2.col(nkc, b2.DECIMAL64, 12, 2, nullable=False), b2.col(nkc + 1, b2.DECIMAL64, 12, 2, nullable=False)
    prog = b2.Program(exprs + [pr * (one - di)])
    spec = [(b2.AGG_SUM, nkc, b2.DECIMAL128, 4, 36)]
    keys_ref, sums, _, _, _ = _reference(k0, price * (100 - disc))
    return b2.Table.from_columns(cols), prog, list(range(nkc)), spec, (keys_ref, sums)


def _check_q3_like(out, nk, ref):
    keys_ref, sums = ref
    got = _by_key(out, nk)
    assert np.array_equal(got[0], keys_ref)
    if nk >= 2:
        assert np.array_equal(got[1], (8000 + keys_ref % 2557).astype(np.int32))
    assert [int(x) for x in got[nk]] == [int(x) for x in sums]


@pytest.mark.parametrize("n", [1_300_007, 2_400_001])
@pytest.mark.parametrize("shape", ["sum_count_1key", "dec128_2keys", "minmax_2keys"])
def test_fused_first_pass_matches_references(b2, shape, n):
    """10 or 11 hash bits (the fused pass, then one 2- or 3-bit pass) for the specialised kernel; the generic kernel's smaller
    table needs one bit more"""
    g = n // 3 + 1
    k0 = _keys(n, g)
    v = np.random.default_rng(n).integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    if shape == "dec128_2keys":
        t, prog, keys, spec, ref = _q3_like(b2, n, g, 2, n)
        call = lambda: b2.scan_aggregate(prog, False, t, keys, spec)
    else:
        k1 = (k0 % 2557).astype(np.int32)
        t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(k1), b2.Column.from_numpy(v)])
        if shape == "sum_count_1key":
            call = lambda: b2.groupby(t, [0], [(b2.AGG_SUM, 2, b2.INT64, 0, 0), (b2.AGG_COUNT, 2, b2.INT64, 0, 0)])
        else:
            call = lambda: b2.groupby(t, [0, 1], [(b2.AGG_MIN, 2, b2.INT64, 0, 0), (b2.AGG_MAX, 2, b2.INT64, 0, 0)])
        keys_ref, sums, cnts, mins, maxs = _reference(k0, v)
    results = []
    for fused in (True, False):
        out, ran = _run(b2, call, fused)
        if shape == "minmax_2keys":
            assert "radix_agg_kernel" in ran, ran
        else:
            assert {"radix_agg_kernel", "radix_agg_fixed_kernel"} & set(ran), ran
        _assert_path(ran, fused, 2)
        if shape == "dec128_2keys":
            _check_q3_like(out, 2, ref)
            got = _by_key(out, 2)
        else:
            got = _by_key(out, 1 if shape == "sum_count_1key" else 2)
            assert np.array_equal(got[0], keys_ref)
            if shape == "sum_count_1key":
                assert np.array_equal(got[1], sums) and np.array_equal(got[2], cnts)
            else:
                assert np.array_equal(got[1], (keys_ref % 2557).astype(np.int32))
                assert np.array_equal(got[2], mins) and np.array_equal(got[3], maxs)
        results.append(got)
    for a, b in zip(*results):
        assert np.array_equal(a, b)


def test_fused_first_pass_with_two_more_passes(b2):
    """17 hash bits (the generic kernel's 2048-slot table at 54 M rows): the fused pass, then an 8-bit and a 1-bit pass.
    Values are the row numbers, so each group's MIN, MAX and COUNT follow from its key: the rows of key k are
    i = i0 + j * G with i0 = k * A^-1 mod G"""
    n = 54_000_001
    g = 27_000_011
    k0 = _keys(n, g)
    t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(np.arange(n, dtype=np.int64))])
    del k0
    specs = [(b2.AGG_MIN, 1, b2.INT64, 0, 0), (b2.AGG_MAX, 1, b2.INT64, 0, 0), (b2.AGG_COUNT, 1, b2.INT64, 0, 0)]
    keys = np.arange(g, dtype=np.int64)
    i0 = (keys * pow(A, -1, g)) % g
    cnt = (n - 1 - i0) // g + 1
    for fused in (True, False):
        out, ran = _run(b2, lambda: b2.groupby(t, [0], specs), fused)
        assert "radix_agg_kernel" in ran, ran
        _assert_path(ran, fused, 3)
        got = _by_key(out, 1)
        assert np.array_equal(got[0], keys)
        assert np.array_equal(got[1], i0) and np.array_equal(got[2], i0 + (cnt - 1) * g) and np.array_equal(got[3], cnt)


def test_predicate_keeps_the_separate_path(b2):
    """a fused predicate compacts the rows, so the materialisation keeps radix_rows_kernel with the switch off too"""
    n = 2_400_001
    g = n // 3 + 1
    k0 = _keys(n, g)
    v = np.random.default_rng(3).integers(-1000, 1000, n, dtype=np.int64)
    t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(v)])
    c0, c1 = b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.INT64, nullable=False)
    prog = b2.Program([c1 >= b2.lit(-500, b2.INT64), c0, c1])
    keep = v >= -500
    keys_ref, sums, _, _, _ = _reference(k0[keep], v[keep])
    out, ran = _run(b2, lambda: b2.scan_aggregate(prog, True, t, [0], [(b2.AGG_SUM, 1, b2.INT64, 0, 0)]), True)
    assert "radix_rows_kernel" in ran and not FUSED & set(ran), ran
    got = _by_key(out, 1)
    assert np.array_equal(got[0], keys_ref) and np.array_equal(got[1], sums)


def test_q3_regime_twice_identical(b2):
    """q3's shape: three key columns in two words, SUM(price * (1 - disc)) as DECIMAL128, 3.6 M groups from 9 M rows;
    the fused path twice (identical results) and the separate path once, all equal to the exact reference"""
    n, g = 9_000_001, 3_600_007
    t, prog, keys, spec, ref = _q3_like(b2, n, g, 3, 33)
    call = lambda: b2.scan_aggregate(prog, False, t, keys, spec)
    runs = []
    for fused in (True, True, False):
        out, ran = _run(b2, call, fused)
        assert "radix_agg_fixed_kernel" in ran, ran
        _assert_path(ran, fused, 2)
        _check_q3_like(out, 3, ref)
        runs.append(_by_key(out, 3))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert np.array_equal(a, b)
