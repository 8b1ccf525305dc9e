"""Every row-moving path against the exact references of tests/movement_reference.py: gather (csrc/gather.cu), slice,
concat and Table.partition (csrc/hash.cu), compared bit for bit at the shapes where the kernels change regime: partial
ballot words, the 64-column launch limit, unaligned validity offsets, the 4096-row tile of the direct partition, the radix
path's 1-, 2- and 4-byte digits and the 8 columns the partition kernel scatters itself."""
import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_hash as H
from tests import movement_reference as M

pytestmark = pytest.mark.gpu
TYPES = M.FIXED_TYPES + [O.STRING]


def _check_table(b2, got_t, exp_cols, what, payload="valid", nullability=True):
    got = M.from_table(b2, got_t)
    assert len(got) == len(exp_cols), what
    for i, (g, e) in enumerate(zip(got, exp_cols)):
        M.assert_same(g, e, "%s col %d" % (what, i), payload=payload, nullability=nullability)


def _imap(b2, idx):
    return b2.Column.from_numpy(np.asarray(idx, np.int32))


# ---- gather -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4097])
def test_gather_every_width(b2, n):
    rng = np.random.default_rng(n)
    src = 3000
    cols = [M.rand_col(rng, dt, src, null_frac=0.3 if k % 2 else 0.0) for k, dt in enumerate(TYPES)]
    gmap = rng.integers(0, src, n)
    if n:
        gmap[: min(n, 2)] = [src - 1, 0][: min(n, 2)]
    got = b2.gather(M.to_table(b2, cols), _imap(b2, gmap))
    _check_table(b2, got, [M.gather(c, gmap, False) for c in cols], "gather n=%d" % n)


@pytest.mark.parametrize("n", [1, 31, 33, 4097])
def test_gather_nullify_out_of_bounds(b2, n):
    """OOB rows (negative, INT32_MIN, src_rows) come back NULL with a zero payload, whether or not the input is nullable"""
    rng = np.random.default_rng(100 + n)
    src = 500
    cols = [M.rand_col(rng, dt, src, null_frac=0.25 if k % 2 else 0.0) for k, dt in enumerate(TYPES)]
    gmap = rng.integers(-2, src + 2, n)
    edges = np.array([-1, M.INT32_MIN, src, src - 1, 0, 2**31 - 1])
    k = min(n, len(edges))
    gmap[rng.choice(n, k, replace=False)] = edges[:k]
    got = b2.gather(M.to_table(b2, cols), _imap(b2, gmap), True)
    # payload="all": the zero bytes of an OOB row are part of the contract (a NULL in-range row keeps its source bytes)
    _check_table(b2, got, [M.gather(c, gmap, True) for c in cols], "gather nullify n=%d" % n, payload="all")


def test_gather_seventy_columns(b2):
    """70 fixed-width columns: the fused kernel takes 64 per launch, so the last 6 go in a second launch"""
    rng = np.random.default_rng(7)
    cols = [M.rand_fixed(rng, M.FIXED_TYPES[k % len(M.FIXED_TYPES)], 700, null_frac=0.2 if k % 3 == 0 else 0.0) for k in range(70)]
    gmap = rng.integers(-5, 705, 1000)
    got = b2.gather(M.to_table(b2, cols), _imap(b2, gmap), True)
    _check_table(b2, got, [M.gather(c, gmap, True) for c in cols], "gather 70 cols", payload="all")


def test_gather_strings_with_no_chars(b2):
    rng = np.random.default_rng(8)
    s = M.rand_strings(rng, 300, null_frac=0.3)
    empty_or_null = np.flatnonzero((np.diff(s.offsets) == 0))
    gmap = rng.choice(empty_or_null, 100)
    got = b2.gather(M.to_table(b2, [s]), _imap(b2, gmap))
    exp = M.gather(s, gmap, False)
    assert len(exp.chars) == 0
    _check_table(b2, got, [exp], "strings without chars")
    got = b2.gather(M.to_table(b2, [s]), _imap(b2, np.full(50, -1)), True)   # every row OOB
    _check_table(b2, got, [M.gather(s, np.full(50, -1), True)], "all OOB strings")


# ---- slice --------------------------------------------------------------------------------------------------------------------
def test_slice_bit_offsets(b2):
    rng = np.random.default_rng(9)
    n = 300
    cols = [M.rand_col(rng, dt, n, null_frac=0.4 if k % 2 else 0.0) for k, dt in enumerate(TYPES)]
    t = M.to_table(b2, cols)
    for start in (0, 1, 7, 8, 31, 32, 33):
        for end in (start, start + 1, start + 40, n):
            got = b2.slice_table(t, start, end)
            assert got.num_rows == end - start
            _check_table(b2, got, [M.slice_col(c, start, end) for c in cols], "slice [%d, %d)" % (start, end))
    with pytest.raises(b2.B2Error):
        b2.slice_table(t, 5, n + 1)
    with pytest.raises(b2.B2Error):
        b2.slice_table(t, 6, 5)


# ---- concat -------------------------------------------------------------------------------------------------------------------
def test_concat_unaligned_parts(b2):
    """row counts that are not multiples of 8 or 32, zero-row parts at the front, in the middle and at the end, nullable and
    non-nullable parts mixed (the result is nullable iff some part is)"""
    rng = np.random.default_rng(10)
    sizes = [0, 13, 1, 0, 45, 7, 100, 33, 0]
    for nullable_parts in ([1, 4, 6], [], [7]):
        parts = [[M.rand_col(rng, dt, sz, null_frac=0.35 if k in nullable_parts else 0.0) for dt in TYPES]
                 for k, sz in enumerate(sizes)]
        got = b2.concat([M.to_table(b2, p) for p in parts])
        exp = [M.concat([p[i] for p in parts]) for i in range(len(TYPES))]
        _check_table(b2, got, exp, "concat nullable parts %s" % nullable_parts)


def test_concat_strings_without_chars_and_decimal128(b2):
    rng = np.random.default_rng(11)
    parts = []
    for sz in (5, 0, 9, 40):
        s = M.rand_strings(rng, sz, null_frac=0.3, empty_frac=1.0)
        parts.append([s, M.rand_fixed(rng, O.DECIMAL128, sz, null_frac=0.2)])
    got = b2.concat([M.to_table(b2, p) for p in parts])
    exp = [M.concat([p[i] for p in parts]) for i in range(2)]
    assert len(exp[0].chars) == 0
    _check_table(b2, got, exp, "concat no chars")


def test_concat_rejects_mismatched_parts(b2):
    rng = np.random.default_rng(12)
    a = M.to_table(b2, [M.rand_fixed(rng, O.INT32, 10), M.rand_fixed(rng, O.INT64, 10)])
    b = M.to_table(b2, [M.rand_fixed(rng, O.INT32, 10), M.rand_fixed(rng, O.FLOAT64, 10)])
    c = M.to_table(b2, [M.rand_fixed(rng, O.INT32, 10)])
    s = M.to_table(b2, [M.rand_fixed(rng, O.INT32, 10), M.rand_strings(rng, 10)])
    for bad in ([a, b], [a, c], [c, a], [a, s]):
        with pytest.raises(b2.B2Error):
            b2.concat(bad)


# ---- partition ----------------------------------------------------------------------------------------------------------------
def _partition_cols(rng, n):
    """11 non-null fixed-width columns of every width (the direct path's kernel scatters the first 8 itself, 16-byte ones
    included; the rest go through the gather map), a nullable column among them and a STRING column"""
    cols = [M.rand_fixed(rng, O.DECIMAL128, n)] + [M.rand_fixed(rng, M.FIXED_TYPES[k], n) for k in range(10)]
    cols.insert(3, M.rand_fixed(rng, O.DECIMAL128, n, null_frac=0.3))
    cols.append(M.rand_strings(rng, n, null_frac=0.2))
    cols.append(M.rand_fixed(rng, O.DECIMAL128, n))
    return cols


def _check_partition(b2, cols, pids, nparts, what):
    out, offs = b2.partition_by_ids(M.to_table(b2, cols), b2.Column.from_numpy(np.asarray(pids, np.int32)), nparts)
    order, eoffs = M.stable_partition(pids, nparts)
    assert offs == eoffs, what
    _check_table(b2, out, [M.take(c, order) for c in cols], what)


@pytest.mark.parametrize("nparts", [1, 2, 1024])
@pytest.mark.parametrize("n", [4095, 4096, 4097, 3 * 4096 + 1])
def test_partition_either_side_of_the_tile(b2, n, nparts):
    """n < 4096 takes the radix path, n >= 4096 with <= 1024 partitions the direct tile path"""
    rng = np.random.default_rng(n * 7 + nparts)
    cols = _partition_cols(rng, n)
    _check_partition(b2, cols, rng.integers(0, nparts, n), nparts, "n=%d nparts=%d" % (n, nparts))


@pytest.mark.parametrize("nparts", [200, 256, 257, 1025, 65536, 65537, 2**20])
def test_partition_radix_digits(b2, nparts):
    """more than 1024 partitions (or fewer than 4096 rows): a radix sort of the ids with 1-, 2- or 4-byte digits.  The ids
    are drawn so that they differ above the low byte (and, past 65536, above the low two bytes)."""
    rng = np.random.default_rng(nparts)
    for n in (3000, 9000):
        cols = _partition_cols(rng, n)
        pids = rng.integers(0, nparts, n)
        pids[: 8] = [0, nparts - 1, nparts // 2, 255 % nparts, 256 % nparts, 65535 % nparts, 65536 % nparts, 1]
        _check_partition(b2, cols, pids, nparts, "n=%d nparts=%d" % (n, nparts))


@pytest.mark.parametrize("n", [1, 2000, 10000])
def test_partition_skew(b2, n):
    rng = np.random.default_rng(n + 3)
    cols = _partition_cols(rng, n)
    for nparts in (1, 5, 1024, 5000):
        _check_partition(b2, cols, np.full(n, nparts - 1), nparts, "all in the last of %d" % nparts)
        _check_partition(b2, cols, rng.choice([0, nparts // 2], n), nparts, "two of %d" % nparts)


def test_partition_empty_table(b2):
    rng = np.random.default_rng(13)
    for nparts in (1, 7, 2000):
        _check_partition(b2, _partition_cols(rng, 0), np.zeros(0, np.int64), nparts, "empty, %d parts" % nparts)


@pytest.mark.parametrize("n", [100, 5000])
def test_partition_rejects_out_of_range_ids(b2, n):
    rng = np.random.default_rng(n)
    t = M.to_table(b2, [M.rand_fixed(rng, O.INT64, n), M.rand_strings(rng, n)])
    for nparts in (3, 1024, 70000):
        for bad in (-1, nparts, M.INT32_MIN, 2**31 - 1):
            pids = rng.integers(0, nparts, n).astype(np.int32)
            pids[n // 2] = bad
            with pytest.raises(b2.B2Error):
                b2.partition_by_ids(t, b2.Column.from_numpy(pids), nparts)
    with pytest.raises(b2.B2Error):
        b2.partition_by_ids(t, b2.Column.from_numpy(np.zeros(n, np.int32)), 0)


@pytest.mark.parametrize("nparts", [1, 7, 1024, 3000])
@pytest.mark.parametrize("n", [2000, 4096 + 100])
def test_hash_partition_two_keys_one_nullable(b2, n, nparts):
    rng = np.random.default_rng(n + nparts)
    k0 = M.rand_fixed(rng, O.INT64, n)
    k0.data[:] = np.frombuffer(rng.integers(0, 300, n).astype(np.int64).tobytes(), np.uint8).reshape(n, 8)
    k1 = M.rand_fixed(rng, O.INT32, n, null_frac=0.3)
    cols = [k0, M.rand_strings(rng, n, null_frac=0.1), k1, M.rand_fixed(rng, O.FLOAT64, n)]
    out, offs = b2.hash_partition(M.to_table(b2, cols), [0, 2], nparts)
    pids = H.partition_ids([M.ocol_of_raw(k0), M.ocol_of_raw(k1)], nparts)
    order, eoffs = M.stable_partition(pids, nparts)
    assert offs == eoffs
    _check_table(b2, out, [M.take(c, order) for c in cols], "hash partition n=%d nparts=%d" % (n, nparts))
