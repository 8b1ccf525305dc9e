"""The radix-partitioned group-by at millions of groups, beyond what test_fullsize_gpu covers:
 * exact sums whose per-group totals cross 2^64 and whose 32-bit pieces carry on about half the rows, through the specialised
   kernel (it keeps its accumulators as 32-bit words and rebuilds the 64- / 128- / 192-bit sums when a table is flushed),
   checked against Python integers;
 * shapes the specialised kernel does not take (MIN, a nullable value column), so the generic kernel stays under test.
Each test checks from the kernel timings which of the two aggregation kernels ran."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, NGROUPS = 6_000_000, 2_000_003


def _keys(rng):
    k0 = rng.integers(0, NGROUPS, N, dtype=np.int64)
    k1 = (k0 % 2557).astype(np.int32)                   # functionally dependent second key: two packed key words
    return k0, k1


def _group_starts(k0):
    order = np.argsort(k0, kind="stable")
    sk = k0[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    return order, sk[starts], starts


def _exact_sums(pieces, order, starts):
    """per-group exact sums of values given as int64 pieces with weights 2^(32 j): each piece sum is exact in int64"""
    tot = np.zeros(len(starts), dtype=object)
    for j, p in enumerate(pieces):
        tot = tot + np.add.reduceat(p[order], starts).astype(object) * (1 << (32 * j))
    return tot


def _sorted_out(out, ngroups_present):
    assert out.num_rows == ngroups_present
    g = out.column(0).to_numpy()[0]
    o = np.argsort(g)
    return g, o


def _radix_kernels(b2, fn):
    """run fn() with kernel timing on; -> (its result, the set of radix aggregation kernels it launched)"""
    b2.profile_enable(True)
    try:
        r = fn()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return r, names & {"radix_agg_kernel", "radix_agg_fixed_kernel"}


@pytest.mark.parametrize("nk", [1, 2])
@pytest.mark.parametrize("kind", ["int64", "dec64", "dec128"])
def test_radix_groupby_exact_sums_with_carries(b2, kind, nk):
    """One SUM per group (q3's plan shape) through the specialised kernel, with one or two packed key words: INT64 (wrapping
    64-bit result), DECIMAL64 (two limbs) and DECIMAL128 (three limbs) over values of both signs near +-2^62 (+-2^100 for
    DECIMAL128), their low 32 bits random so that the low word carries on about half the rows.  A third of the groups hold only
    positive values, a third only negative ones, the rest both, so exact totals pass +-2^64 (+-2^102)."""
    rng = np.random.default_rng({"int64": 9001, "dec64": 9008, "dec128": 9016}[kind] + nk)
    k0, k1 = _keys(rng)
    cls = k0 % 3
    sign = np.where(cls == 0, 1, np.where(cls == 1, -1, np.where(rng.random(N) < 0.5, 1, -1))).astype(np.int64)
    mag = (1 << 62) - rng.integers(0, 1 << 40, N, dtype=np.int64)
    lo32 = rng.integers(0, 1 << 32, N, dtype=np.int64)
    if kind != "dec128":
        val = sign * ((mag & ~np.int64(0xFFFFFFFF)) | lo32)
        col = b2.Column.from_numpy(val, dtype=b2.INT64) if kind == "int64" else b2.Column.from_numpy(val, dtype=b2.DECIMAL64, scale=2)
        pieces = [val & np.int64(0xFFFFFFFF), val >> np.int64(32)]
    else:
        # v = sign * (mag * 2^38 + lo32): |v| < 2^100, given to the column as (lo, hi) 64-bit words
        hi_mag = mag >> np.int64(26)                                        # mag * 2^38 = hi_mag * 2^64 + (mag % 2^26) * 2^38
        lo_mag = ((mag & np.int64((1 << 26) - 1)) << np.int64(38)) | lo32
        lo_u = lo_mag.view(np.uint64)
        neg = sign < 0
        lo_w = np.where(neg, (~lo_u) + np.uint64(1), lo_u)
        hi_w = np.where(neg, (~hi_mag.view(np.uint64)) + (lo_u == 0).astype(np.uint64), hi_mag.view(np.uint64))
        col = b2.Column.from_numpy(np.stack([lo_w, hi_w], axis=1), dtype=b2.DECIMAL128, scale=2)
        lw, hw = lo_w.view(np.int64), hi_w.view(np.int64)
        pieces = [lw & np.int64(0xFFFFFFFF), (lw >> np.int64(32)) & np.int64(0xFFFFFFFF), hw & np.int64(0xFFFFFFFF), hw >> np.int64(32)]
    t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(k1), col])
    order, present, starts = _group_starts(k0)
    want = _exact_sums(pieces, order, starts)
    assert max(abs(int(x)) for x in want) > (1 << (102 if kind == "dec128" else 64))   # the totals do leave 64 (102) bits
    if kind == "int64":
        want = [((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63) for x in want]          # Spark's long sum wraps
        spec = (b2.AGG_SUM, 2, b2.INT64, 0, 0)
    else:
        spec = (b2.AGG_SUM, 2, b2.DECIMAL128, 2, 38)
    keys = [0, 1][:nk]
    out, ran = _radix_kernels(b2, lambda: b2.groupby(t, keys, [spec]))
    assert ran == {"radix_agg_fixed_kernel"}
    g, o = _sorted_out(out, len(present))
    assert np.array_equal(g[o], present)
    if nk == 2:
        assert np.array_equal(out.column(1).to_numpy()[0][o], (present % 2557).astype(np.int32))
    vals, valid = out.column(nk).to_numpy()
    assert valid.all()
    assert [int(x) for x in vals[o]] == [int(x) for x in want]


@pytest.mark.parametrize("shape", ["min", "nullable_sum"])
def test_radix_groupby_generic_kernel_shapes(b2, shape):
    """high-cardinality shapes outside the specialised kernel: MIN, and a SUM over a nullable column (all-NULL groups give NULL)"""
    rng = np.random.default_rng(77 if shape == "min" else 78)
    k0, k1 = _keys(rng)
    val = rng.integers(-10_000_000, 10_000_000, N, dtype=np.int64)
    order, present, starts = _group_starts(k0)
    if shape == "min":
        t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(k1), b2.Column.from_numpy(val)])
        out, ran = _radix_kernels(b2, lambda: b2.groupby(t, [0, 1], [(b2.AGG_MIN, 2, b2.INT64, 0, 0), (b2.AGG_SUM, 2, b2.INT64, 0, 0)]))
        assert ran == {"radix_agg_kernel"}
        g, o = _sorted_out(out, len(present))
        assert np.array_equal(g[o], present)
        assert np.array_equal(out.column(2).to_numpy()[0][o], np.minimum.reduceat(val[order], starts))
        assert np.array_equal(out.column(3).to_numpy()[0][o], np.add.reduceat(val[order], starts))
    else:
        valid = rng.random(N) < 0.6
        t = b2.Table.from_columns([b2.Column.from_numpy(k0), b2.Column.from_numpy(k1), b2.Column.from_numpy(val, valid=valid)])
        out, ran = _radix_kernels(b2, lambda: b2.groupby(t, [0, 1], [(b2.AGG_SUM, 2, b2.INT64, 0, 0), (b2.AGG_COUNT, 2, b2.INT64, 0, 0)]))
        assert ran == {"radix_agg_kernel"}
        g, o = _sorted_out(out, len(present))
        assert np.array_equal(g[o], present)
        vv = np.where(valid, val, 0)[order]
        cnt = np.add.reduceat(valid[order].astype(np.int64), starts)
        sums, svalid = out.column(2).to_numpy()
        assert np.array_equal(svalid[o], cnt > 0)
        assert np.array_equal(sums[o][cnt > 0], np.add.reduceat(vv, starts)[cnt > 0])
        assert np.array_equal(out.column(3).to_numpy()[0][o], cnt)
