"""Every accumulation path of the hash aggregate against exact integer references, at the edges where the
accumulators go wrong: decimal SUM at the result-precision boundary (DECIMAL64 and DECIMAL128 results), totals past
2^128, mixed-sign carries, nullable sums, a fused predicate at high cardinality, many key shapes and MIN/MAX of the
extreme values.  The paths and how each test reaches them:
 * keyless          b2.reduce: private per-thread accumulators, then the CTA combine
 * smem_few         keyed, <= 1 M rows, <= 4 groups in every 32-row slice: the REDUX-per-group mode of the CTA table
 * smem_lane        keyed, <= 1 M rows, 60 groups in random order: every lane updates its own slot
 * global           <= 1 M rows and 120 K groups (the CTA tables overflow), or inputs the radix path refuses
 * radix            > 1 M rows, high cardinality, a plan outside the specialised kernel's shapes (SUM + COUNT of a decimal)
 * radix_fixed      > 1 M rows, high cardinality, NOT NULL SUM only: the specialised kernel
Each test asserts from the kernel timings which aggregation kernel ran.  References are vectorised: per-group sums of
32-bit pieces with np.add.reduceat, exact as Python ints, pinned to the oracle on a small instance first."""
import numpy as np
import pytest

from oracle import spark_cpu as O

pytestmark = pytest.mark.gpu

KERNELS = {"aggregate_smem_kernel", "aggregate_global_kernel", "radix_agg_kernel", "radix_agg_fixed_kernel"}
PATHS = ["keyless", "smem_few", "smem_lane", "global", "radix", "radix_fixed"]
# (filler rows, filler groups) per path
GEOMETRY = {"keyless": (100_000, 1), "smem_few": (100_000, 3), "smem_lane": (60_000, 60), "global": (250_000, 120_000),
            "radix": (2_100_000, 700_000), "radix_fixed": (2_100_000, 700_000)}
M64 = (1 << 64) - 1


def _ran(b2, fn):
    """run fn() with kernel timing on; -> (its result, the set of aggregation kernels it launched)"""
    b2.profile_enable(True)
    try:
        r = fn()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return r, names & KERNELS


def _assert_path(path, ran):
    if path == "global":
        assert "aggregate_global_kernel" in ran and not ran & {"radix_agg_kernel", "radix_agg_fixed_kernel"}, ran
    else:
        want = {"keyless": "aggregate_smem_kernel", "smem_few": "aggregate_smem_kernel", "smem_lane": "aggregate_smem_kernel",
                "radix": "radix_agg_kernel", "radix_fixed": "radix_agg_fixed_kernel"}[path]
        assert ran == {want}, (path, ran)


# ---- exact references ------------------------------------------------------------------------------------------
def _words(vals):
    """python ints (|v| < 2^127) -> (lo, hi) int64 arrays of their two's-complement 64-bit words"""
    lo = np.array([((int(v) & M64) ^ (1 << 63)) - (1 << 63) for v in vals], dtype=np.int64)
    hi = np.array([int(v) >> 64 for v in vals], dtype=np.int64)
    return lo, hi


def exact_group_sums(g, lo, hi, valid):
    """per-group (sorted ids, exact sums as python ints, valid counts) of the 128-bit values hi * 2^64 + (lo as unsigned);
    each 32-bit piece sums exactly in int64"""
    order = np.argsort(g, kind="stable")
    sg = g[order]
    starts = np.flatnonzero(np.r_[True, sg[1:] != sg[:-1]]) if len(g) else np.zeros(0, np.int64)
    v = valid[order].astype(np.int64)
    m = np.int64(0xFFFFFFFF)
    pieces = [lo & m, (lo >> np.int64(32)) & m, hi & m, hi >> np.int64(32)]
    tot = np.zeros(len(starts), dtype=object)
    for j, p in enumerate(pieces):
        tot = tot + np.add.reduceat(p[order] * v, starts).astype(object) * (1 << (32 * j)) if len(starts) else tot
    cnt = np.add.reduceat(v, starts) if len(starts) else np.zeros(0, np.int64)
    return sg[starts], tot, cnt


def decimal_result(tot, cnt, p):
    """Spark's decimal SUM result: NULL for an empty group or when |total| >= 10^p (GpuCheckOverflowAfterSum)"""
    ok = np.array([c > 0 and abs(int(t)) < 10 ** p for t, c in zip(tot, cnt)], dtype=bool)
    return [int(t) if o else None for t, o in zip(tot, ok)]


def test_exact_reference_is_pinned_to_the_oracle():
    rng = np.random.default_rng(5)
    n = 3000
    g = rng.integers(0, 40, n)
    vals = [int(x) for x in rng.integers(-2**62, 2**62, n)]
    vals = [v * (1 << 40) if i % 3 == 0 else v for i, v in enumerate(vals)]                      # some reach ~2^102
    vals[:8] = [10**37 * 9] * 8
    g[:8] = 3                                                                                    # group 3 overflows 10^38
    valid = rng.random(n) < 0.8
    valid[:8] = True
    valid[g == 7] = False                                                                        # an all-NULL group
    lo, hi = _words(vals)
    keys, tot, cnt = exact_group_sums(g, lo, hi, valid)
    cols = [O.OCol(g.astype(np.int64), np.ones(n, bool), (O.INT64, 0, 0)), O.OCol(np.array(vals, dtype=object), valid, (O.DECIMAL128, 38, 0))]
    exp = O.groupby_cols(cols, [0], [(O.AGG_SUM, 1, O.DECIMAL128, 0, 38), (O.AGG_COUNT, 1)])
    want = dict(zip(exp[0].to_pylist(), zip(exp[1].to_pylist(), exp[2].to_pylist())))
    assert want == dict(zip(keys.tolist(), zip(decimal_result(tot, cnt, 38), cnt.tolist())))
    assert any(v is None for v, c in want.values() if c > 0) and any(v is None for v, c in want.values() if c == 0)
    red = O.reduce_cols([cols[1]], [(O.AGG_SUM, 0, O.DECIMAL128, 0, 38)])[0].to_pylist()[0]
    _, t1, c1 = exact_group_sums(np.zeros(n, np.int64), lo, hi, valid)
    assert decimal_result(t1, c1, 38) == [red]


# ---- inputs ----------------------------------------------------------------------------------------------------
def layout(rng, path, specials, filler, valid_frac=1.0):
    """-> (group id per row, lo, hi, valid).  Special group i (a list of python ints) has id i.  The filler rows get
    `filler(rng, n)` -> (lo, hi); on keyless / smem_few they fall into the special groups (so filler must be zero there
    when specials are given), elsewhere into GEOMETRY's own groups.  Row order is random."""
    nrows, ngroups = GEOMETRY[path]
    if path in ("keyless", "smem_few") and specials:
        assert len(specials) <= (1 if path == "keyless" else 4)
        gf = rng.integers(0, len(specials), nrows)
    else:
        gf = len(specials) + rng.integers(0, ngroups, nrows)
    sv = [v for grp in specials for v in grp]
    gs = np.array([i for i, grp in enumerate(specials) for _ in grp], dtype=np.int64)
    slo, shi = _words(sv) if sv else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    flo, fhi = filler(rng, nrows)
    g = np.concatenate([gs, gf])
    lo, hi = np.concatenate([slo, flo]), np.concatenate([shi, fhi])
    valid = np.ones(len(g), bool)
    if valid_frac < 1.0:
        valid[len(gs):] = rng.random(nrows) < valid_frac
    perm = rng.permutation(len(g))
    g, lo, hi, valid = g[perm], lo[perm], hi[perm], valid[perm]
    if path == "smem_few":      # the REDUX mode needs <= 4 groups in each 32-row slice
        assert len(np.unique(g)) <= 4
    if path == "smem_lane":     # ... and the per-lane mode more than 4 in most of them
        s = g[: len(g) // 32 * 32].reshape(-1, 32)
        assert np.mean([len(np.unique(r)) > 4 for r in s[:200]]) > 0.9
    return g, lo, hi, valid


def zero_filler(rng, n):
    return np.zeros(n, np.int64), np.zeros(n, np.int64)


def small_filler(rng, n):
    lo = rng.integers(-1000, 1000, n, dtype=np.int64)
    return lo, lo >> np.int64(63)


def carry_filler(bits):
    """values of both signs near +-2^bits (bits = 62 or 100) with random low 32 bits: the low words carry on about half
    the additions, and the groups' totals cross 2^64 (2^102)"""
    def f(rng, n):
        sign = np.where(rng.random(n) < 0.5, 1, -1).astype(np.int64)
        mag = (1 << 62) - rng.integers(0, 1 << 40, n, dtype=np.int64)
        lo32 = rng.integers(0, 1 << 32, n, dtype=np.int64)
        if bits == 62:
            v = sign * ((mag & ~np.int64(0xFFFFFFFF)) | lo32)
            return v, v >> np.int64(63)
        hi_mag = mag >> np.int64(24)                                     # mag * 2^40 = hi_mag * 2^64 + (mag % 2^24) * 2^40
        lo_mag = (((mag & np.int64((1 << 24) - 1)) << np.int64(40)) | lo32).view(np.uint64)
        neg = sign < 0
        lo = np.where(neg, (~lo_mag) + np.uint64(1), lo_mag).view(np.int64)
        hi = np.where(neg, ~hi_mag + (lo_mag == 0).astype(np.int64), hi_mag)
        return lo, hi
    return f


def key_of(g):
    """the INT64 key of group id g: negative and positive, spread over all 64 bits"""
    with np.errstate(over="ignore"):
        return (g.astype(np.int64) * np.int64(-7046029254386353131)) ^ np.int64(0x5DEECE66D)


def value_column(b2, lo, hi, valid, dtype, scale):
    v = None if valid.all() else valid
    if dtype == b2.DECIMAL128:
        return b2.Column.from_numpy(np.stack([lo.view(np.uint64), hi.view(np.uint64)], axis=1), dtype=dtype, scale=scale, valid=v)
    return b2.Column.from_numpy(lo, dtype=dtype, scale=scale, valid=v)


def run_sum(b2, path, g, lo, hi, valid, dtype, scale, p, out_dtype, monkeypatch=None):
    """SUM (and, on the generic radix path, COUNT) of the value column per group, checked against the exact reference;
    -> the output table"""
    val = value_column(b2, lo, hi, valid, dtype, scale)
    spec = (b2.AGG_SUM, 1, out_dtype, scale, p)
    specs = [spec, (b2.AGG_COUNT, 1)] if path == "radix" or not valid.all() else [spec]
    if path == "keyless":
        t = b2.Table.from_columns([b2.Column.from_numpy(np.zeros(len(g), np.int64)), val])
        out, ran = _ran(b2, lambda: b2.reduce(t, specs))
        keys, tot, cnt = exact_group_sums(np.zeros(len(g), np.int64), lo, hi, valid)
        got_k = keys
        o = np.arange(1)
        first = 0
    else:
        t = b2.Table.from_columns([b2.Column.from_numpy(key_of(g)), val])
        out, ran = _ran(b2, lambda: b2.groupby(t, [0], specs))
        keys, tot, cnt = exact_group_sums(g, lo, hi, valid)
        assert out.num_rows == len(keys)
        got_k = out.column(0).to_numpy()[0]
        o = np.argsort(got_k)
        ko = np.argsort(key_of(keys))
        keys, tot, cnt = keys[ko], tot[ko], cnt[ko]
        assert np.array_equal(got_k[o], key_of(keys))
        first = 1
    _assert_path(path, ran)
    vals, ok = out.column(first).to_numpy()
    want = decimal_result(tot, cnt, p)
    assert np.array_equal(ok[o], np.array([w is not None for w in want])), "validity differs"
    assert [int(x) for x, k in zip(vals[o], ok[o]) if k] == [w for w in want if w is not None]
    if len(specs) == 2:
        assert np.array_equal(out.column(first + 1).to_numpy()[0][o], cnt)
    return out


def _split(total, lim, parts):
    """`parts` python ints, each of magnitude < lim, that add up to total"""
    q = total // parts
    xs = [q] * (parts - 1) + [total - q * (parts - 1)]
    assert all(abs(x) < lim for x in xs) and sum(xs) == total
    return xs


# ---- 1. decimal SUM at the precision boundary -------------------------------------------------------------------
# p = 38: DECIMAL128(38,0) in, DECIMAL128 out; p = 22: DECIMAL128(22,2) in and out (a Final merge's shape);
# p = 17: DECIMAL64(17,2) in and out, a DECIMAL64 result (a DECIMAL32 column cannot reach 10^17 in a test-sized input)
BOUNDARY = {38: ("DECIMAL128", 0, "DECIMAL128"), 22: ("DECIMAL128", 2, "DECIMAL128"), 17: ("DECIMAL64", 2, "DECIMAL64")}


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("p", [38, 22, 17])
def test_decimal_sum_at_precision_boundary(b2, path, p):
    """groups whose exact totals are 10^p - 1, 10^p, -(10^p - 1), -10^p: value, NULL, value, NULL"""
    rng = np.random.default_rng(100 + p)
    dt, scale, odt = BOUNDARY[p]
    lim = 10 ** p
    totals = [lim - 1, lim, -(lim - 1), -lim]
    groups = [_split(tt, lim, 3) for tt in totals]
    filler = zero_filler if path in ("keyless", "smem_few") else small_filler
    for grp in ([[x] for x in groups] if path == "keyless" else [groups]):
        g, lo, hi, valid = layout(rng, path, grp, filler)
        out = run_sum(b2, path, g, lo, hi, valid, getattr(b2, dt), scale, p, getattr(b2, odt))
        if path != "keyless":
            k = out.column(0).to_numpy()[0]
            vals, ok = out.column(1).to_numpy()
            got = {int(kk): (int(v) if o else None) for kk, v, o in zip(k, vals, ok)}
            assert [got[int(key_of(np.array([i]))[0])] for i in range(4)] == [lim - 1, None, -(lim - 1), None]


# ---- 2. totals past 128 bits ------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
def test_decimal_sum_past_128_bits(b2, path):
    """exact totals 2^128 + 5 and -2^128 - 5 (three values of 10^38 - 1 plus a remainder below 10^38): their low 128 bits
    are +-5; 2^128 - 7 and -2^128 + 7: the low 128 bits are in range but of the wrong sign.  All four are NULL."""
    rng = np.random.default_rng(200)
    big = 10 ** 38 - 1
    groups = []
    for tt in [(1 << 128) + 5, -(1 << 128) - 5, (1 << 128) - 7, -(1 << 128) + 7]:
        s = 1 if tt > 0 else -1
        rest = tt - 3 * s * big
        assert abs(rest) < 10 ** 38
        groups.append([s * big, s * big, s * big, rest])
    filler = zero_filler if path in ("keyless", "smem_few") else small_filler
    for grp in ([[x] for x in groups] if path == "keyless" else [groups]):
        g, lo, hi, valid = layout(rng, path, grp, filler)
        out = run_sum(b2, path, g, lo, hi, valid, b2.DECIMAL128, 0, 38, b2.DECIMAL128)
        vals, ok = out.column(0 if path == "keyless" else 1).to_numpy()
        assert (~ok).sum() >= len(grp)


# ---- 3. mixed-sign carries --------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("bits", [62, 100])
def test_decimal_sum_mixed_sign_carries(b2, path, bits):
    """DECIMAL64 values near +-2^62 and DECIMAL128 values near +-2^100, random low words, into a DECIMAL128(38) result"""
    rng = np.random.default_rng(300 + bits)
    g, lo, hi, valid = layout(rng, path, [], carry_filler(bits))
    _, tot, _ = exact_group_sums(g, lo, hi, valid)
    assert max(abs(int(x)) for x in tot) > (1 << (bits + 2))                     # the totals do leave 64 (102) bits
    run_sum(b2, path, g, lo, hi, valid, b2.DECIMAL64 if bits == 62 else b2.DECIMAL128, 2, 38, b2.DECIMAL128)


# ---- 4. nullable decimal SUM ------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["smem_lane", "global", "radix"])
def test_nullable_decimal_sum(b2, path):
    """30 % of the filler values NULL, all-NULL groups and one overflowing group: NULL for both, told apart by COUNT"""
    rng = np.random.default_rng(400)
    over = _split(10 ** 38 + 12345, 10 ** 38, 3)
    g, lo, hi, valid = layout(rng, path, [over], carry_filler(100), valid_frac=0.7)
    dead = np.isin(g, np.arange(1, 1 + GEOMETRY[path][1], 17))                  # every 17th filler group: all NULL
    valid[dead] = False
    out = run_sum(b2, path, g, lo, hi, valid, b2.DECIMAL128, 2, 38, b2.DECIMAL128)
    vals, ok = out.column(1).to_numpy()
    cnt = out.column(2).to_numpy()[0]
    assert ((~ok) & (cnt == 0)).sum() > 0 and ((~ok) & (cnt > 0)).sum() == 1


# ---- 8. the same radix-eligible input through the specialised kernel and the global table ------------------------
def test_specialised_kernel_agrees_with_global_table(b2, monkeypatch):
    rng = np.random.default_rng(800)
    g, lo, hi, valid = layout(rng, "radix_fixed", [], carry_filler(100))
    a = run_sum(b2, "radix_fixed", g, lo, hi, valid, b2.DECIMAL128, 2, 38, b2.DECIMAL128)
    monkeypatch.setenv("B2_AGG_NO_RADIX", "1")
    b = run_sum(b2, "global", g, lo, hi, valid, b2.DECIMAL128, 2, 38, b2.DECIMAL128)
    ka, kb = a.column(0).to_numpy()[0], b.column(0).to_numpy()[0]
    oa, ob = np.argsort(ka), np.argsort(kb)
    assert np.array_equal(ka[oa], kb[ob])
    assert list(a.column(1).to_numpy()[0][oa]) == list(b.column(1).to_numpy()[0][ob])


# ---- 5. fused predicate at high cardinality ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def pred_input():
    rng = np.random.default_rng(500)
    n = 3_000_000
    g = rng.integers(0, 1_000_000, n)
    lo, hi = carry_filler(62)(rng, n)
    sel = rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)
    return g, lo, hi, sel


@pytest.mark.parametrize("keep", ["half", "none", "all"])
def test_fused_predicate_high_cardinality(b2, pred_input, keep):
    """b2.scan_aggregate with the predicate fused: sel < 0 keeps about half the rows, sel > INT32_MAX none, sel >= INT32_MIN all"""
    g, lo, hi, sel = pred_input
    t = b2.Table.from_columns([b2.Column.from_numpy(key_of(g)), b2.Column.from_numpy(lo, dtype=b2.DECIMAL64, scale=2),
                               b2.Column.from_numpy(sel)])
    c = b2.col(2, b2.INT32, nullable=False)
    pred = {"half": c < b2.lit(0, b2.INT32), "none": c > b2.lit(2**31 - 1, b2.INT32), "all": c >= b2.lit(-2**31, b2.INT32)}[keep]
    prog = b2.Program([pred, b2.col(0, b2.INT64, nullable=False), b2.col(1, b2.DECIMAL64, 18, 2, nullable=False)])
    specs = [(b2.AGG_SUM, 1, b2.DECIMAL128, 2, 38), (b2.AGG_COUNT_ALL, 0)]
    out, ran = _ran(b2, lambda: b2.scan_aggregate(prog, True, t, [0], specs))
    m = {"half": sel < 0, "none": np.zeros(len(g), bool), "all": np.ones(len(g), bool)}[keep]
    if keep == "none":      # the cardinality probe sees no group, so the shared-memory table takes it: no group at all
        assert out.num_rows == 0 and ran == {"aggregate_smem_kernel"}
        return
    assert ran == {"radix_agg_kernel"}                       # a fused predicate tracks validity: the generic kernel
    keys, tot, cnt = exact_group_sums(g[m], lo[m], hi[m], np.ones(int(m.sum()), bool))
    assert out.num_rows == len(keys)
    gk = out.column(0).to_numpy()[0]
    o, ko = np.argsort(gk), np.argsort(key_of(keys))
    assert np.array_equal(gk[o], key_of(keys)[ko])
    vals, ok = out.column(1).to_numpy()
    assert ok.all() and [int(x) for x in vals[o]] == [int(x) for x in tot[ko]]
    assert np.array_equal(out.column(2).to_numpy()[0][o], cnt[ko])


# ---- 6. key shapes at high cardinality --------------------------------------------------------------------------
NK = 2_000_000


def _float_keys(rng, g):
    """finite keys per group, and groups 0..3 made of NaN payload variants, +-0.0, +inf, -inf"""
    k = np.where(g % 2 == 0, 1.0, -1.0) * (g.astype(np.float64) * 0.37 + 1.0)
    nans = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)
    k[g == 0] = nans[rng.integers(0, 4, int((g == 0).sum()))]
    k[g == 1] = np.array([0.0, -0.0])[rng.integers(0, 2, int((g == 1).sum()))]
    k[g == 2], k[g == 3] = np.inf, -np.inf
    return k


def _norm_float(k):
    k = k.copy()
    k[k == 0] = 0.0
    k[np.isnan(k)] = np.nan
    return k


def _key_shape(b2, rng, shape, g):
    """-> (key columns, a function from group ids to the expected key arrays, the path)"""
    with np.errstate(over="ignore"):
        k64 = key_of(g)
    if shape == "i32_i64_i16_i8":    # 15 bytes; the INT64 straddles the two packed key words (bits 32..95)
        f = lambda x: [(-(x % 100_003)).astype(np.int32), key_of(x), ((x % 65_536) - 32_768).astype(np.int16), ((x % 256) - 128).astype(np.int8)]
        dts, path = [b2.INT32, b2.INT64, b2.INT16, b2.INT8], "radix"
    elif shape == "date_dec64":
        f = lambda x: [(x % 40_000 - 20_000).astype(np.int32), key_of(x)]
        dts, path = [b2.DATE32, b2.DECIMAL64], "radix"
    elif shape == "bool_i64":
        f = lambda x: [(x % 2).astype(np.int8), key_of(x)]
        dts, path = [b2.BOOL8, b2.INT64], "radix"
    elif shape == "i64_i64":         # exactly 16 bytes
        f = lambda x: [key_of(x), -key_of(x) - 1]
        dts, path = [b2.INT64, b2.INT64], "radix"
    elif shape == "i64_i64_i8":      # 17 bytes: the global table
        f = lambda x: [key_of(x), -key_of(x) - 1, (x % 3 - 1).astype(np.int8)]
        dts, path = [b2.INT64, b2.INT64, b2.INT8], "global"
    else:
        raise AssertionError(shape)
    cols = [b2.Column.from_numpy(a, dtype=d, scale=2 if d == b2.DECIMAL64 else 0) for a, d in zip(f(g), dts)]
    return cols, f, path


@pytest.fixture(scope="module")
def key_input():
    rng = np.random.default_rng(600)
    g = rng.integers(0, 600_000, NK)
    v = rng.integers(-10**12, 10**12, NK, dtype=np.int64)
    return rng, g, v


def _check_keyed(out, nk, want_keys, sums, cnts):
    """output key columns equal want_keys once both are sorted by all keys; then the SUM and COUNT columns"""
    got = [out.column(i).to_numpy()[0] for i in range(nk)]
    o, wo = np.lexsort(got[::-1]), np.lexsort(want_keys[::-1])
    for a, b in zip(got, want_keys):
        assert np.array_equal(a[o], b[wo])
    assert np.array_equal(out.column(nk).to_numpy()[0][o], sums[wo])
    assert np.array_equal(out.column(nk + 1).to_numpy()[0][o], cnts[wo])


def _int_sums(g, v):
    order = np.argsort(g, kind="stable")
    sg = g[order]
    starts = np.flatnonzero(np.r_[True, sg[1:] != sg[:-1]])
    return sg[starts], np.add.reduceat(v[order], starts), np.diff(np.r_[starts, len(g)])


@pytest.mark.parametrize("shape", ["i32_i64_i16_i8", "date_dec64", "bool_i64", "i64_i64", "i64_i64_i8"])
def test_key_shapes_high_cardinality(b2, key_input, monkeypatch, shape):
    rng, g, v = key_input
    cols, f, path = _key_shape(b2, rng, shape, g)
    nk = len(cols)
    t = b2.Table.from_columns(cols + [b2.Column.from_numpy(v)])
    out, ran = _ran(b2, lambda: b2.groupby(t, list(range(nk)), [(b2.AGG_SUM, nk, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]))
    _assert_path(path if path == "global" else "radix_fixed", ran)
    keys, sums, cnts = _int_sums(g, v)
    assert out.num_rows == len(keys)
    _check_keyed(out, nk, f(keys), sums, cnts)


@pytest.mark.parametrize("shape", ["float64", "nullable_i64", "string"])
def test_key_shapes_special_values(b2, key_input, shape):
    """FLOAT64 keys (NaN payloads one group, +-0.0 one group) on the radix path; nullable INT64 keys (NULL its own group)
    and STRING keys mixing lengths that pack into 8 bytes with longer ones, which take the global table above 1 M rows"""
    rng, g, v = key_input
    if shape == "float64":
        k = _float_keys(rng, g)
        t = b2.Table.from_columns([b2.Column.from_numpy(k), b2.Column.from_numpy(v)])
        want_path = "radix_fixed"
    elif shape == "nullable_i64":
        kv = g != 5                                                          # group 5 is the NULL key
        t = b2.Table.from_columns([b2.Column.from_numpy(key_of(g), valid=kv), b2.Column.from_numpy(v)])
        want_path = "global"
    else:
        ids = np.unique(g)
        strs = [(b"%x" % i) if i % 3 else (b"long-key-%09d" % i) for i in ids.tolist()]   # 1..5 bytes pack, 18 do not
        lens = np.array([len(s) for s in strs], dtype=np.int64)
        pos = np.searchsorted(ids, g)
        offs = np.zeros(NK + 1, np.int64)
        offs[1:] = np.cumsum(lens[pos])
        pool = np.frombuffer(b"".join(strs), dtype=np.uint8)
        pstart = np.r_[0, np.cumsum(lens)[:-1]]
        idx = np.repeat(pstart[pos] - offs[:-1], lens[pos]) + np.arange(offs[-1])
        t = b2.Table.from_columns([b2.Column.from_string_buffers(pool[idx], offs.astype(np.int32)), b2.Column.from_numpy(v)])
        want_path = "global"
    out, ran = _ran(b2, lambda: b2.groupby(t, [0], [(b2.AGG_SUM, 1, b2.INT64, 0, 0), (b2.AGG_COUNT_ALL, 0)]))
    _assert_path(want_path, ran)
    gk, gv = out.column(0).to_numpy()
    if shape == "float64":     # one group per id: the NaN variants all belong to id 0 and +-0.0 to id 1
        keys, sums, cnts = _int_sums(g, v)
        assert out.num_rows == len(keys)
        want = _norm_float(_float_keys(rng, keys))
        o, wo = np.argsort(_norm_float(gk)), np.argsort(want)
        assert np.array_equal(_norm_float(gk)[o], want[wo], equal_nan=True)
    elif shape == "nullable_i64":
        keys, sums, cnts = _int_sums(g, v)
        assert out.num_rows == len(keys)
        got = np.where(gv, gk, np.iinfo(np.int64).min)
        want = np.where(keys != 5, key_of(keys), np.iinfo(np.int64).min)
        assert (~gv).sum() == 1
        o, wo = np.argsort(got), np.argsort(want)
        assert np.array_equal(got[o], want[wo])
    else:
        keys, sums, cnts = _int_sums(g, v)
        assert out.num_rows == len(keys)
        back = np.array([int(s[9:]) if s.startswith(b"long-key-") else int(s, 16) for s in gk.tolist()], dtype=np.int64)
        o, wo = np.argsort(back), np.argsort(keys)
        assert np.array_equal(back[o], keys[wo])
    assert np.array_equal(out.column(1).to_numpy()[0][o], sums[wo])
    assert np.array_equal(out.column(2).to_numpy()[0][o], cnts[wo])


# ---- 7. MIN / MAX of extreme values -----------------------------------------------------------------------------
MINMAX_TYPES = {"i8_i16": [("INT8", np.int8), ("INT16", np.int16)], "i32_i64": [("INT32", np.int32), ("INT64", np.int64)],
                 "dec32_dec64": [("DECIMAL32", np.int32), ("DECIMAL64", np.int64)], "float": []}


@pytest.mark.parametrize("path,types", [(p, t) for p in ["smem_lane", "global", "radix"] for t in MINMAX_TYPES if (p, t) != ("radix", "float")])
def test_min_max_extremes(b2, path, types):
    """group 0 holds only the type's minimum, group 1 only its maximum, group 2 both (they equal the accumulators'
    initial values); FLOAT32 / FLOAT64 groups of NaN only, +-0.0 only, +inf only, -inf only, +-inf.  The radix path takes
    integers only, at most five value columns (MIN and MAX of one column are two), so two types per run."""
    rng = np.random.default_rng(700 + len(types) + len(path))
    nrows, ngroups = GEOMETRY[path]
    nrows = min(nrows, 1_200_000)
    g = np.concatenate([np.repeat(np.arange(6), 5), 6 + rng.integers(0, ngroups, nrows)])
    rng.shuffle(g)
    cols, arrays = [b2.Column.from_numpy(key_of(g))], []
    for name, npt in MINMAX_TYPES[types]:
        info = np.iinfo(npt)
        a = rng.integers(info.min, info.max, len(g), endpoint=True, dtype=np.int64).astype(npt)
        a[g == 0], a[g == 1] = info.min, info.max
        a[g == 2] = np.where(rng.random(int((g == 2).sum())) < 0.5, info.min, info.max)
        arrays.append(a)
        cols.append(b2.Column.from_numpy(a, dtype=getattr(b2, name)))
    if types == "float":
        for npt in (np.float32, np.float64):
            a = rng.standard_normal(len(g)).astype(npt)
            m = {0: np.nan, 2: np.inf, 3: -np.inf}
            for gi, x in m.items():
                a[g == gi] = x
            a[g == 1] = np.array([0.0, -0.0], dtype=npt)[rng.integers(0, 2, int((g == 1).sum()))]
            a[g == 5] = np.array([np.inf, -np.inf], dtype=npt)[rng.integers(0, 2, int((g == 5).sum()))]
            arrays.append(a)
            cols.append(b2.Column.from_numpy(a))
    t = b2.Table.from_columns(cols)
    specs = [(kind, 1 + i, 0, 0, 0) for i in range(len(arrays)) for kind in (b2.AGG_MIN, b2.AGG_MAX)]
    out, ran = _ran(b2, lambda: b2.groupby(t, [0], specs))
    _assert_path(path, ran)
    order = np.argsort(g, kind="stable")
    sg = g[order]
    starts = np.flatnonzero(np.r_[True, sg[1:] != sg[:-1]])
    gk = out.column(0).to_numpy()[0]
    o, wo = np.argsort(gk), np.argsort(key_of(sg[starts]))
    assert np.array_equal(gk[o], key_of(sg[starts])[wo])
    for i, a in enumerate(arrays):
        s = a[order]
        if a.dtype.kind == "f":     # Spark: NaN is the greatest value, -0.0 == 0.0
            isn = np.isnan(s)
            mn = np.fmin.reduceat(np.where(isn, np.inf, s), starts)
            mn[np.logical_and.reduceat(isn, starts)] = np.nan
            mx = np.maximum.reduceat(s, starts)
        else:
            mn, mx = np.minimum.reduceat(s, starts), np.maximum.reduceat(s, starts)
        gmn, gmx = out.column(1 + 2 * i).to_numpy()[0][o], out.column(2 + 2 * i).to_numpy()[0][o]
        assert np.array_equal(gmn, mn[wo], equal_nan=a.dtype.kind == "f"), (i, a.dtype)
        assert np.array_equal(gmx, mx[wo], equal_nan=a.dtype.kind == "f"), (i, a.dtype)
        if a.dtype.kind != "f":
            info = np.iinfo(a.dtype)
            first = {int(k): j for j, k in enumerate(sg[starts][wo])}
            assert (gmn[first[0]], gmx[first[0]], gmn[first[1]], gmx[first[1]]) == (info.min, info.min, info.max, info.max)
