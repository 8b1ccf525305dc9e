"""Every path that orders rows (sort.cu over the normalised key of sortkey.cuh) against the exact rank-based reference of
tests/sort_reference.py: the one-CTA bitonic sort and the LSD radix sort, top-N by radix select and its fallbacks, the
merge-path merge of sorted runs, lower / upper bound, and the GpuSortExec / GpuTopN operators.  Permutations and output
columns are compared exactly, floats bit for bit (so -0.0 and 0.0 stay apart in the output and NaN payloads survive).
Inputs sit at the edges of the normalised key: type extremes and signs, every class of float, strings with NUL and high
bytes, shared 8-byte prefixes and the 1024-byte limit, DECIMAL128 words.  Which kernel ran shows in the kernel timings."""
import numpy as np
import pytest

from oracle import spark_cpu as O
from spark_rapids_b200 import execs as E
from tests import datagen as G
from tests import sort_reference as S

pytestmark = pytest.mark.gpu

ORDERS = [(1, 1), (1, 0), (0, 1), (0, 0)]   # (ascending, nulls_first)
SMALL, RADIX, MERGE, BOUNDS = "small_sort_kernel", "radix_scatter_kernel", "merge_path_kernel", "bounds_kernel"
TOPN_HIST, TOPN_PREFIX, TOPN_MASK = "topn_hist8_kernel", "hist_prefix_kernel", "topn_mask_kernel"
ERR_INVALID, ERR_UNSUPPORTED = 1, 5
SELECT_MIN_ROWS = 1 << 18
TOPN_ROWS = 300_000

INT_BITS = {O.INT8: 8, O.INT16: 16, O.INT32: 32, O.INT64: 64, O.DATE32: 32, O.TIMESTAMP_US: 64}
DEC_PREC = {O.DECIMAL32: 9, O.DECIMAL64: 18, O.DECIMAL128: 38}
NP = {O.BOOL8: np.int8, O.INT8: np.int8, O.INT16: np.int16, O.INT32: np.int32, O.INT64: np.int64, O.DATE32: np.int32,
      O.TIMESTAMP_US: np.int64, O.FLOAT32: np.float32, O.FLOAT64: np.float64}
FIXED_TYPES = [(O.BOOL8, 0, 0), (O.INT8, 0, 0), (O.INT16, 0, 0), (O.INT32, 0, 0), (O.INT64, 0, 0), (O.FLOAT32, 0, 0), (O.FLOAT64, 0, 0),
               (O.DATE32, 0, 0), (O.TIMESTAMP_US, 0, 0), (O.DECIMAL32, 9, 2), (O.DECIMAL64, 18, 2), (O.DECIMAL128, 38, 2)]
ALL_TYPES = FIXED_TYPES + [(O.STRING, 0, 0)]


TYPE_NAMES = ["bool8", "int8", "int16", "int32", "int64", "float32", "float64", "date32", "timestamp", "decimal32", "decimal64", "decimal128",
              "string"]


def tid(typ):
    return TYPE_NAMES[typ[0]]


# ---- inputs ------------------------------------------------------------------------------------------------------------
def float_edges(dt):
    if dt == O.FLOAT32:
        bits = [0x7f800000, 0xff800000, 0x00000000, 0x80000000, 0x7f7fffff, 0xff7fffff, 0x00800000, 0x80800000, 0x00000001, 0x80000001,
                0x7fc00000, 0x7f800001, 0x7fffffff, 0xffc00000, 0xff800001, 0x3f800000, 0xbf800000]
        return np.array(bits, np.uint32).view(np.float32)
    bits = [0x7ff0000000000000, 0xfff0000000000000, 0, 0x8000000000000000, 0x7fefffffffffffff, 0xffefffffffffffff, 0x0010000000000000,
            0x8010000000000000, 1, 0x8000000000000001, 0x7ff8000000000000, 0x7ff0000000000001, 0x7fffffffffffffff, 0xfff8000000000000,
            0xfff0000000000001, 0x3ff0000000000000, 0xbff0000000000000]
    return np.array(bits, np.uint64).view(np.float64)


def decimal128_edges():
    lim = 10**38 - 1
    out = [lim, -lim, lim - 1, -lim + 1, -1, 0, 1, 2**63 - 1, 2**63, -2**63, -2**63 - 1, 2**64 - 1, 2**64, 2**64 + 1, -2**64, -2**64 + 1,
           -2**64 - 1]
    for hi in (12345, -12345, 0, -1):   # same high word, low words apart in their top and bottom bits
        out += [(hi << 64) + lo for lo in (0, 1, 2**63 - 1, 2**63, 2**64 - 1, 0x0100000000000000)]
    return out


STRING_EDGES = [b"", b"\0", b"\0\0", b"a", b"a\0", b"a\0\0", b"ab", b"a\0b", b"\x7f", b"\x80", b"\xff", b"\xff\xff", b"\x7f\xff", b"\x80\0",
                "é".encode(), "日本語".encode(), "😀".encode(), b"abcdefg", b"abcdefg\0", b"abcdefgh", b"abcdefgh\0", b"abcdefghi", b"abcdefgha",
                b"abcdefgz", b"abcdefhh", b"abcdefghij\xff", b"abcdefghh", b"x" * 1023, b"x" * 1024, b"x" * 1022 + b"y", b"x" * 1023 + b"\0",
                b"y" + b"\0" * 1022, b"\0" * 1024]


def edge_values(rng, typ, n):
    """n values of `typ`: the type's edges, each several times, mixed with random values (numpy / object array)"""
    dt = typ[0]
    half = n // 2
    if dt == O.BOOL8:
        return rng.integers(0, 2, n).astype(np.int8)
    if dt in INT_BITS:
        b = INT_BITS[dt]
        lo, hi = -2**(b - 1), 2**(b - 1) - 1
        edges = np.array([lo, lo + 1, -2, -1, 0, 1, 2, hi - 1, hi, -(1 << (b - 2)), 1 << (b - 2)], np.int64)
        rnd = np.concatenate([rng.integers(lo, hi, n - half, endpoint=True, dtype=np.int64), rng.integers(-30, 30, half)])
        v = np.where(rng.random(n) < 0.3, edges[rng.integers(0, len(edges), n)], rnd)
        return v.astype(NP[dt])
    if dt in (O.FLOAT32, O.FLOAT64):
        edges = float_edges(dt)
        rnd = np.concatenate([rng.standard_normal(n - half) * 10.0 ** rng.integers(-40, 38, n - half), np.round(rng.standard_normal(half) * 4)])
        with np.errstate(over="ignore"):   # float32 overflow: more infinities
            rnd = rnd.astype(NP[dt])
        pick = rng.random(n) < 0.3
        v = rnd.copy()
        v[pick] = edges[rng.integers(0, len(edges), int(pick.sum()))]
        return v
    if dt in DEC_PREC:
        lim = 10**DEC_PREC[dt] - 1
        if dt == O.DECIMAL128:
            edges = decimal128_edges()
            rnd = [int(h) * 2**64 + int(lo) for h, lo in zip(rng.integers(-3, 3, n), rng.integers(0, 2**63, n))]
            rnd = [r if i % 3 else int(x) for i, (r, x) in enumerate(zip(rnd, rng.integers(-50, 50, n)))]
        else:
            edges = [lim, -lim, lim - 1, -lim + 1, -1, 0, 1]
            rnd = [int(x) for x in rng.integers(-lim, lim, n, endpoint=True, dtype=np.int64)]
            rnd = [r if i % 3 else int(x) for i, (r, x) in enumerate(zip(rnd, rng.integers(-50, 50, n)))]
        pick = rng.random(n) < 0.3
        e = rng.integers(0, len(edges), n)
        return np.array([edges[e[i]] if pick[i] else rnd[i] for i in range(n)], dtype=object)
    assert dt == O.STRING
    alphabet = [0, 1, 0x41, 0x61, 0x62, 0x7f, 0x80, 0xc3, 0xa9, 0xff]
    lens = rng.integers(0, 14, n)
    prefixes = [b"", b"abcdefg", b"abcdefgh", b"abcdefghi"]
    pick = rng.random(n) < 0.3
    e = rng.integers(0, len(STRING_EDGES), n)
    pre = rng.integers(0, len(prefixes), n)
    return np.array([STRING_EDGES[e[i]] if pick[i] else prefixes[pre[i]] + bytes(rng.choice(alphabet, lens[i]).astype(np.uint8).tolist())
                     for i in range(n)], dtype=object)


def edge_col(rng, typ, n, null_frac=0.1):
    valid = rng.random(n) >= null_frac if null_frac > 0 else np.ones(n, bool)
    return O.OCol(edge_values(rng, typ, n), valid, typ)


def few_col(rng, typ, n, k, null_frac=0.1):
    """values of a k-value set (many ties), edges included"""
    pool = edge_values(rng, typ, max(k, 2))[:k]
    vals = pool[rng.integers(0, k, n)] if pool.dtype != object else np.array([pool[i] for i in rng.integers(0, k, n)], dtype=object)
    valid = rng.random(n) >= null_frac if null_frac > 0 else np.ones(n, bool)
    return O.OCol(vals, valid, typ)


def index_col(n, base=0):
    return O.OCol(np.arange(base, base + n, dtype=np.int32), np.ones(n, bool), (O.INT32, 0, 0))


def take(cols, idx):
    return [O.OCol(c.values[idx], c.valid[idx], c.typ) for c in cols]


def table(b2, cols):
    return G.to_b2_table(b2, cols)


def profiled(b2, fn):
    """-> (fn(), {kernel timer name: launches})"""
    b2.profile_enable(True)
    try:
        out = fn()
        names = {k["name"]: k["launches"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return out, names


def set_path(monkeypatch, path):
    if path == "radix":
        monkeypatch.setenv("B2_SORT_NO_SMALL", "1")
    else:
        monkeypatch.delenv("B2_SORT_NO_SMALL", raising=False)


def assert_cols(got_table, cols, idx, what=""):
    """the device table equals the reference columns gathered by idx, floats bit for bit"""
    idx = np.asarray(idx, np.int64)
    assert got_table.num_rows == len(idx), (what, got_table.num_rows, len(idx))
    for i, c in enumerate(cols):
        vals, valid = got_table.column(i).to_numpy()
        ev = c.valid[idx]
        assert np.array_equal(valid, ev), (what, i, np.flatnonzero(valid != ev)[:10])
        exp = c.values[idx]
        dt = c.typ[0]
        if dt in (O.FLOAT32, O.FLOAT64):
            u = np.uint32 if dt == O.FLOAT32 else np.uint64
            assert np.array_equal(vals[ev].view(u), np.asarray(exp, NP[dt])[ev].view(u)), (what, i)
        elif exp.dtype == object or vals.dtype == object:
            g = [bytes(x) if dt == O.STRING else int(x) for x in vals[ev]]
            e = [bytes(x) if dt == O.STRING else int(x) for x in exp[ev]]
            bad = [k for k in range(len(g)) if g[k] != e[k]]
            assert not bad, (what, i, bad[:5])
        else:
            assert np.array_equal(vals[ev].astype(np.int64), np.asarray(exp[ev]).astype(np.int64)), (what, i)


def sort_and_check(b2, cols, keys, path_kernel, what=""):
    """b2_sort_order and b2_order_by against the reference; asserts the sort kernel that ran"""
    t = table(b2, cols)
    perm, names = profiled(b2, lambda: b2.sort_order(t, keys).to_numpy()[0])
    exp = S.sort_order(cols, keys)
    assert np.array_equal(perm.astype(np.int64), exp), (what, keys, np.flatnonzero(perm != exp)[:10])
    if path_kernel is None:
        assert SMALL not in names and RADIX not in names, names
    else:
        other = RADIX if path_kernel == SMALL else SMALL
        assert path_kernel in names and other not in names, (what, names)
    assert_cols(b2.order_by(t, keys), cols, exp, what)
    return names


# ---- sort: edge values of every type on both paths -----------------------------------------------------------------------
@pytest.mark.parametrize("path", ["small", "radix"])
@pytest.mark.parametrize("typ", ALL_TYPES, ids=tid)
def test_sort_edge_values(b2, typ, path, monkeypatch):
    set_path(monkeypatch, path)
    rng = np.random.default_rng(typ[0] * 2 + (path == "radix"))
    n = 3000
    cols = [edge_col(rng, typ, n), index_col(n)]
    for asc, nf in ORDERS:
        sort_and_check(b2, cols, [(0, asc, nf)], SMALL if path == "small" else RADIX, (tid(typ), asc, nf))


@pytest.mark.parametrize("path", ["small", "radix"])
def test_sort_all_null_and_no_validity_columns(b2, path, monkeypatch):
    """an all-NULL key (null byte only decides nothing; input order stays) and keys without a validity buffer (no null byte)"""
    set_path(monkeypatch, path)
    rng = np.random.default_rng(5)
    n = 2000
    all_null = [O.OCol(edge_values(rng, t, n), np.zeros(n, bool), t) for t in ((O.INT32, 0, 0), (O.STRING, 0, 0), (O.FLOAT64, 0, 0))]
    no_valid = [edge_col(rng, t, n, null_frac=0) for t in ((O.INT64, 0, 0), (O.FLOAT32, 0, 0), (O.STRING, 0, 0), (O.DECIMAL128, 38, 0))]
    kern = SMALL if path == "small" else RADIX
    for asc, nf in ORDERS:
        for c in all_null:
            names = sort_and_check(b2, [c, index_col(n)], [(0, asc, nf)], None if path == "radix" else kern, "all null")
            if path == "radix":
                assert RADIX not in names and SMALL not in names   # one constant byte: every digit is trivial
        for c in no_valid:
            sort_and_check(b2, [c, index_col(n)], [(0, asc, nf)], kern, "no validity")
        sort_and_check(b2, all_null[:1] + no_valid[:1] + [index_col(n)], [(0, asc, nf), (1, 1 - asc, nf)], kern, "null then value")


def test_string_key_length_limit(b2, monkeypatch):
    """strings up to 1024 bytes sort (1028-byte value key); one of 1025 bytes is refused, also under a NULL elsewhere"""
    for path in ("small", "radix"):
        set_path(monkeypatch, path)
        vals = np.array([b"x" * 1024, b"x" * 1023, b"x" * 1023 + b"\0", b"", b"x" * 1024, b"w" + b"\xff" * 1023], dtype=object)
        c = O.OCol(vals, np.array([True, True, True, True, True, False]), (O.STRING, 0, 0))
        for asc, nf in ORDERS:
            sort_and_check(b2, [c, index_col(6)], [(0, asc, nf)], SMALL if path == "small" else RADIX)
        bad = table(b2, [O.OCol(np.array([b"a", b"y" * 1025], dtype=object), np.ones(2, bool), (O.STRING, 0, 0))])
        for fn in (lambda: b2.sort_order(bad, [(0, 1, 1)]), lambda: b2.top_n(bad, [(0, 1, 1)], 1),
                   lambda: b2.merge_sorted([bad, bad], [(0, 1, 1)])):
            with pytest.raises(b2.B2Error) as e:
                fn()
            assert e.value.code == ERR_UNSUPPORTED


# ---- sort: sizes on each path, and skipped digits -------------------------------------------------------------------------
def size_cols(rng, n):
    return [few_col(rng, (O.INT16, 0, 0), n, 7), edge_col(rng, (O.FLOAT64, 0, 0), n), index_col(n)]


SIZE_KEYS = [(0, 0, 0), (1, 1, 1)]


@pytest.mark.parametrize("n", [0, 1, 2, 3, 8191, 8192, 8193, 16383, 16384, 16385])
def test_sort_sizes_bitonic(b2, n, monkeypatch):
    set_path(monkeypatch, "small")
    cols = size_cols(np.random.default_rng(n), n)
    kern = None if n < 2 else (SMALL if n <= 16384 else RADIX)
    sort_and_check(b2, cols, SIZE_KEYS, kern, n)


@pytest.mark.parametrize("n", [2, 4095, 4096, 4097, 8192, 12289, 16385])
def test_sort_sizes_radix(b2, n, monkeypatch):
    set_path(monkeypatch, "radix")
    cols = size_cols(np.random.default_rng(n + 1), n)
    sort_and_check(b2, cols, SIZE_KEYS, RADIX, n)


def test_radix_skips_trivial_digits(b2, monkeypatch):
    """digits on which every row agrees cost no pass: all keys equal (none), keys that differ in one byte (one pass per
    chunk that holds it), keys that differ only in the top byte of a chunk"""
    set_path(monkeypatch, "radix")
    rng = np.random.default_rng(77)
    n = 20000

    def i64(v):
        return O.OCol(np.asarray(v, np.int64), np.ones(n, bool), (O.INT64, 0, 0))
    base = -0x1234567890abcdef
    cases = [
        ([i64(np.full(n, base))], 0),
        ([i64((base & ~(0xff << 24)) | (rng.integers(0, 256, n) << 24))], 1),
        ([i64(rng.integers(-128, 128, n) << 56)], 1),
        ([i64(np.full(n, 7)), i64(rng.integers(-128, 128, n) << 56)], 1),                # second chunk, top byte
        ([i64(rng.integers(0, 2, n) << 56), i64(rng.integers(0, 2, n) + base)], 2),     # top byte of chunk 0, low byte of chunk 1
    ]
    for cols, passes in cases:
        keys = [(k, 1, 1) for k in range(len(cols))]
        names = sort_and_check(b2, cols + [index_col(n)], keys, RADIX if passes else None)
        assert names.get(RADIX, 0) == passes, (passes, names)
        for asc in (0, 1):   # DESC flips every byte: the same digits are trivial
            names = sort_and_check(b2, cols + [index_col(n)], [(k, asc, 1) for k in range(len(cols))], RADIX if passes else None)
            assert names.get(RADIX, 0) == passes


# ---- sort: several keys --------------------------------------------------------------------------------------------------
KEYSETS = {   # name -> key column types (NULLs or not); the row key's byte length is in the name
    "7B": [((O.INT8, 0, 0), 0), ((O.INT16, 0, 0), 0), ((O.INT32, 0, 0), 0)],
    "8B": [((O.INT8, 0, 0), 0), ((O.INT16, 0, 0), 0), ((O.INT32, 0, 0), 0), ((O.BOOL8, 0, 0), 0)],
    "9B": [((O.INT64, 0, 0), 0), ((O.INT8, 0, 0), 0)],
    "16B": [((O.INT64, 0, 0), 0), ((O.FLOAT64, 0, 0), 0)],
    "17B": [((O.INT64, 0, 0), 0), ((O.INT64, 0, 0), 0), ((O.INT8, 0, 0), 0)],
    "nullable-29B": [((O.INT16, 0, 0), 0.2), ((O.DECIMAL128, 38, 0), 0.1), ((O.DATE32, 0, 0), 0.1), ((O.FLOAT32, 0, 0), 0.1)],
    "string-middle": [((O.INT32, 0, 0), 0.1), ((O.STRING, 0, 0), 0.1), ((O.INT16, 0, 0), 0.1)],
}


@pytest.mark.parametrize("path", ["small", "radix"])
@pytest.mark.parametrize("keyset", list(KEYSETS))
def test_sort_multi_key(b2, keyset, path, monkeypatch):
    """few distinct values per key, so rows tie on the first chunk and later chunks decide; mixed directions and null
    placements"""
    set_path(monkeypatch, path)
    rng = np.random.default_rng(list(KEYSETS).index(keyset) * 2 + (path == "radix"))
    n = 6000
    spec = KEYSETS[keyset]
    cols = [few_col(rng, t, n, 5 if i < len(spec) - 1 else 40, nf) for i, (t, nf) in enumerate(spec)] + [index_col(n)]
    for trial in range(4):
        keys = [(k, int(rng.integers(0, 2)), int(rng.integers(0, 2))) for k in range(len(spec))]
        sort_and_check(b2, cols, keys, SMALL if path == "small" else RADIX, (keyset, keys))


def test_sort_sixteen_keys_and_not_seventeen(b2, monkeypatch):
    rng = np.random.default_rng(16)
    n = 5000
    cols = [few_col(rng, (O.INT8, 0, 0), n, 3, 0.2) for _ in range(17)] + [index_col(n)]
    keys = [(k, k % 2, (k // 2) % 2) for k in range(16)]
    for path in ("small", "radix"):
        set_path(monkeypatch, path)
        sort_and_check(b2, cols, keys, SMALL if path == "small" else RADIX)
    t = table(b2, cols)
    keys17 = keys + [(16, 1, 1)]
    for fn in (lambda: b2.sort_order(t, keys17), lambda: b2.top_n(t, keys17, 3), lambda: b2.merge_sorted([t, t], keys17),
               lambda: b2.search_bounds(t, t, keys17, 0)):
        with pytest.raises(b2.B2Error) as e:
            fn()
        assert e.value.code == ERR_INVALID


# ---- top-N ------------------------------------------------------------------------------------------------------------------
def i64_col(v, valid=None):
    return O.OCol(np.asarray(v, np.int64), np.ones(len(v), bool) if valid is None else valid, (O.INT64, 0, 0))


def topn_check(b2, cols, keys, limit, t=None):
    """b2_top_n against the first `limit` rows of the reference order -> kernel launches"""
    t = t if t is not None else table(b2, cols)
    out, names = profiled(b2, lambda: b2.top_n(t, keys, limit))
    exp = S.top_n(cols, keys, limit)
    assert_cols(out, cols, exp, (keys, limit))
    return names


def test_topn_select_limits(b2):
    """n >= 2^18: limit 1 and n/16 take the radix select; n/16 + 1 sorts everything"""
    rng = np.random.default_rng(301)
    n = TOPN_ROWS
    key = i64_col(rng.integers(-2**63, 2**63 - 1, n, endpoint=True, dtype=np.int64), rng.random(n) >= 0.1)
    cols = [key, index_col(n)]
    t = table(b2, cols)
    for keys in ([(0, 1, 1)], [(0, 0, 0)], [(0, 1, 0)]):
        for limit, selected in ((1, True), (n // 16, True), (n // 16 + 1, False)):
            names = topn_check(b2, cols, keys, limit, t)
            assert TOPN_HIST in names if selected else TOPN_HIST not in names
            assert (TOPN_MASK in names) == selected, (keys, limit, names)


def test_topn_select_ties_and_refinement_rounds(b2):
    """ties around the threshold stay in input order; a first varying digit with more than 8192 rows in the wanted bucket
    takes one refinement round, two such digits two"""
    rng = np.random.default_rng(302)
    n = TOPN_ROWS
    r16 = rng.integers(0, 1 << 16, n)
    cases = [
        ("ties", O.OCol(rng.integers(0, 100, n).astype(np.int32), np.ones(n, bool), (O.INT32, 0, 0)), 4500, 0),
        ("one round", i64_col((rng.integers(0, 4, n) << 16) | r16), 1000, 1),
        ("two rounds", i64_col((rng.integers(0, 4, n) << 24) | (rng.integers(0, 4, n) << 16) | r16), 1000, 2),
        ("two rounds desc", i64_col((rng.integers(0, 4, n) << 24) | (rng.integers(0, 4, n) << 16) | r16), 1000, 2),
    ]
    for what, key, limit, rounds in cases:
        cols = [key, index_col(n)]
        keys = [(0, 0, 0)] if "desc" in what else [(0, 1, 1)]
        names = topn_check(b2, cols, keys, limit)
        assert TOPN_MASK in names, (what, names)
        assert names.get(TOPN_PREFIX, 0) == rounds, (what, names)


def test_topn_select_skips_constant_leading_chunks(b2):
    """every row agrees on the first chunk (the high word of a DECIMAL128) or the first two (a 16-byte common string prefix):
    the selection moves on to the next chunk, one histogram per chunk looked at"""
    rng = np.random.default_rng(303)
    n = TOPN_ROWS
    lo = rng.integers(0, 2**63, n, dtype=np.int64).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64)
    for hi in (12345, -7):
        words = np.stack([lo, np.full(n, np.int64(hi)).view(np.uint64)], axis=1)
        dcol = b2.Column.from_numpy(words, dtype=b2.DECIMAL128, scale=2)
        ref = O.OCol(np.array([(hi << 64) + int(x) for x in lo], dtype=object), np.ones(n, bool), (O.DECIMAL128, 38, 2))
        cols = [ref, index_col(n)]
        t = b2.Table.from_columns([dcol, G.to_b2_column(b2, cols[1])])
        for keys in ([(0, 1, 1)], [(0, 0, 0)]):
            names = topn_check(b2, cols, keys, 100, t)
            assert names.get(TOPN_HIST) == 2 and TOPN_MASK in names, names
    chars = np.empty((n, 24), np.uint8)
    chars[:, :16] = np.frombuffer(b"Customer#0000000", np.uint8)
    chars[:, 16:] = rng.integers(0x30, 0x3a, (n, 8))
    chars[::97, 20:] = 0x30   # ties
    scol = b2.Column.from_string_buffers(chars.ravel(), np.arange(0, 24 * n + 1, 24, dtype=np.int32))
    ref = O.OCol(np.array([r.tobytes() for r in chars], dtype=object), np.ones(n, bool), (O.STRING, 0, 0))
    cols = [ref, index_col(n)]
    t = b2.Table.from_columns([scol, G.to_b2_column(b2, cols[1])])
    for keys in ([(0, 1, 1)], [(0, 0, 1)]):
        names = topn_check(b2, cols, keys, 500, t)
        assert names.get(TOPN_HIST) == 3 and TOPN_MASK in names, names


def test_topn_fallbacks(b2):
    """one value holding most rows (the candidates would pass n/4), n just below 2^18, limit 0, limit above n: a full sort"""
    rng = np.random.default_rng(304)
    n = TOPN_ROWS
    v = rng.integers(-2**31, 2**31 - 1, n).astype(np.int32)
    v[rng.random(n) < 0.7] = -2**31
    cols = [O.OCol(v, rng.random(n) >= 0.01, (O.INT32, 0, 0)), index_col(n)]
    names = topn_check(b2, cols, [(0, 1, 0)], 10)
    assert TOPN_HIST in names and TOPN_MASK not in names, names
    m = SELECT_MIN_ROWS - 1
    cols = [i64_col(rng.integers(-2**63, 2**63 - 1, m, dtype=np.int64)), index_col(m)]
    t = table(b2, cols)
    for limit in (1, 0, m + 5):
        names = topn_check(b2, cols, [(0, 0, 1)], limit, t)
        assert TOPN_HIST not in names and TOPN_MASK not in names, (limit, names)
    small = [edge_col(rng, (O.FLOAT32, 0, 0), 700), index_col(700)]
    for limit in (0, 1, 699, 700, 701, 10**9):
        for asc, nf in ORDERS:
            topn_check(b2, small, [(0, asc, nf)], limit)
    with pytest.raises(b2.B2Error) as e:
        b2.top_n(table(b2, small), [(0, 1, 1)], -1)
    assert e.value.code == ERR_INVALID


@pytest.mark.parametrize("typ", ALL_TYPES, ids=tid)
def test_topn_edge_values(b2, typ):
    rng = np.random.default_rng(typ[0] + 400)
    n = 3000
    cols = [edge_col(rng, typ, n), index_col(n)]
    for asc, nf in ORDERS:
        for limit in (1, 17, 2999):
            topn_check(b2, cols, [(0, asc, nf)], limit)


# ---- merge --------------------------------------------------------------------------------------------------------------------
def sorted_parts(cols, sizes, keys, tag_base=0):
    """`cols` cut into consecutive parts of `sizes` rows, each sorted by `keys` (the reference), each with a tag column
    (part * 100000 + row) so that ties across parts show in the output"""
    parts, a = [], 0
    for p, sz in enumerate(sizes):
        piece = [O.OCol(c.values[a:a + sz], c.valid[a:a + sz], c.typ) for c in cols]
        perm = S.sort_order(piece, keys)
        parts.append(take(piece, perm) + [index_col(sz, (tag_base + p) * 100000)])
        a += sz
    return parts


def merge_check(b2, parts, keys, what=""):
    tabs = [table(b2, p) for p in parts]
    out, names = profiled(b2, lambda: b2.merge_sorted(tabs, keys))
    exp = S.merge(parts, keys)
    assert_cols(out, S.concat(parts), exp, what)
    nonempty = sum(len(p[0].valid) > 0 for p in parts)
    assert (MERGE in names) == (nonempty >= 2), (what, names)
    return names


@pytest.mark.parametrize("typ", ALL_TYPES, ids=tid)
def test_merge_edge_values(b2, typ):
    rng = np.random.default_rng(typ[0] + 500)
    sizes = [700, 0, 2048, 1301]
    c = edge_col(rng, typ, sum(sizes))
    for asc, nf in ORDERS:
        merge_check(b2, sorted_parts([c], sizes, [(0, asc, nf)]), [(0, asc, nf)], (tid(typ), asc, nf))


@pytest.mark.parametrize("sizes", [[1000], [2047, 2049], [2048, 2048], [1, 4096, 3], [0, 2048, 0, 2047, 0], [500, 600, 700, 800, 900],
                                   [0, 0], [4097, 1, 2048, 2049, 2050, 6000, 7]])
def test_merge_runs(b2, sizes):
    """one run, two, an odd number (the carried run), empty runs, runs at the 2048-row tile edge; keys with few values so
    that ties cross runs and must come out in table order"""
    rng = np.random.default_rng(sum(sizes) + len(sizes))
    n = sum(sizes)
    cols = [few_col(rng, (O.INT32, 0, 0), n, 9, 0.1), few_col(rng, (O.STRING, 0, 0), n, 4, 0.1)]
    for keys in ([(0, 1, 1)], [(0, 0, 0), (1, 1, 0)]):
        merge_check(b2, sorted_parts(cols, sizes, keys), keys, (sizes, keys))


def test_merge_first_chunk_ties_resolved_by_later_chunks(b2):
    """the merge compares the first 8 key bytes and computes later chunks only on ties: a constant-ish first key, then keys
    that decide (a string, a DECIMAL128 across chunk boundaries)"""
    rng = np.random.default_rng(601)
    sizes = [3000, 2500, 4100]
    n = sum(sizes)
    cols = [few_col(rng, (O.INT64, 0, 0), n, 2, 0.05), few_col(rng, (O.STRING, 0, 0), n, 30, 0.05), edge_col(rng, (O.DECIMAL128, 38, 0), n)]
    for keys in ([(0, 1, 1), (1, 1, 1), (2, 1, 1)], [(0, 0, 1), (1, 0, 0), (2, 1, 0)], [(0, 1, 0), (2, 0, 0), (1, 1, 1)]):
        merge_check(b2, sorted_parts(cols, sizes, keys), keys, keys)


def test_merge_strings_of_different_longest_length(b2):
    """each table's longest string differs (3, 40 and 1024 bytes): the merge pads every string key to the longest of all"""
    rng = np.random.default_rng(602)
    short = O.OCol(np.array([bytes(rng.choice([0x61, 0x62, 0], rng.integers(0, 4)).astype(np.uint8).tolist()) for _ in range(900)], dtype=object),
                   rng.random(900) > 0.1, (O.STRING, 0, 0))
    mid = O.OCol(np.array([b"ab" + bytes(rng.choice([0x61, 0x62, 0], rng.integers(0, 39)).astype(np.uint8).tolist()) for _ in range(700)],
                          dtype=object), rng.random(700) > 0.1, (O.STRING, 0, 0))
    long = O.OCol(np.array([b"a" * 1024, b"a", b"b" * 1000, b"", b"ab"] * 40, dtype=object), np.ones(200, bool), (O.STRING, 0, 0))
    for asc, nf in ORDERS:
        keys = [(0, asc, nf)]
        parts = []
        for p, c in enumerate((short, mid, long)):
            perm = S.sort_order([c], keys)
            parts.append(take([c], perm) + [index_col(len(perm), p * 100000)])
        merge_check(b2, parts, keys, (asc, nf))
        merge_check(b2, parts[::-1], keys, (asc, nf, "reversed"))


def test_merge_rejects_mixed_decimal_scales(b2):
    """regression: b2_merge_sorted concatenated DECIMAL64 scale 2 and scale 4 inputs and compared their unscaled integers"""
    a = b2.Table.from_columns([b2.Column.from_numpy(np.array([100, 250], np.int64), dtype=b2.DECIMAL64, scale=2)])
    b = b2.Table.from_columns([b2.Column.from_numpy(np.array([10000, 25000], np.int64), dtype=b2.DECIMAL64, scale=4)])
    for fn in (lambda: b2.merge_sorted([a, b], [(0, 1, 1)]), lambda: b2.concat([a, b])):
        with pytest.raises(b2.B2Error) as e:
            fn()
        assert e.value.code == ERR_INVALID
    c = b2.Table.from_columns([b2.Column.from_numpy(np.array([300], np.int64), dtype=b2.DECIMAL64, scale=2)])
    assert b2.merge_sorted([a, c], [(0, 1, 1)]).column(0).to_pylist() == [100, 250, 300]


# ---- lower / upper bound ----------------------------------------------------------------------------------------------------
def probe_values(rng, c, n):
    """present values, their neighbours, and fresh edge values (NULLs included)"""
    dt = c.typ[0]
    ok = np.flatnonzero(c.valid)
    pres = c.values[rng.choice(ok, n // 3)] if len(ok) else edge_values(rng, c.typ, n // 3)
    if dt == O.BOOL8:
        nb = (1 - pres).astype(pres.dtype)
    elif dt in (O.FLOAT32, O.FLOAT64):
        with np.errstate(over="ignore", invalid="ignore"):   # max -> inf, NaN -> NaN
            nb = np.nextafter(pres, np.where(rng.random(len(pres)) < 0.5, np.inf, -np.inf).astype(pres.dtype))
    elif pres.dtype == object:
        nb = np.array([int(x) + int(d) for x, d in zip(pres, rng.choice([-1, 1], len(pres)))], dtype=object)
    else:
        nb = (pres.astype(np.int64) + rng.choice([-1, 1], len(pres))).astype(pres.dtype)
    fresh = edge_values(rng, c.typ, n - 2 * (n // 3))
    vals = np.concatenate([pres, nb, fresh]) if pres.dtype != object else np.array(list(pres) + list(nb) + list(fresh), dtype=object)
    return O.OCol(vals, rng.random(len(vals)) >= 0.1, c.typ)


def bounds_check(b2, sc, pc, keys, what=""):
    st, pt = table(b2, sc), table(b2, pc)
    for upper in (False, True):
        got, names = profiled(b2, lambda: b2.search_bounds(st, pt, keys, upper).to_numpy()[0])
        exp = S.bounds(sc, pc, keys, upper)
        assert np.array_equal(got.astype(np.int64), exp), (what, keys, upper, np.flatnonzero(got != exp)[:10])
        if len(pc[0].valid):
            assert BOUNDS in names, names


@pytest.mark.parametrize("typ", FIXED_TYPES, ids=tid)
def test_search_bounds_edge_values(b2, typ):
    rng = np.random.default_rng(typ[0] + 700)
    c = edge_col(rng, typ, 2500)
    for asc, nf in ORDERS:
        keys = [(0, asc, nf)]
        sc = take([c], S.sort_order([c], keys))
        pc = [probe_values(rng, c, 900)]
        bounds_check(b2, sc, pc, keys, (tid(typ), asc, nf))
    if typ[0] in (O.FLOAT32, O.FLOAT64):   # NaN, -0.0 and 0.0 probes against a table holding all three
        z = O.OCol(np.array([-1.0, -0.0, 0.0, -0.0, np.nan, np.inf, np.nan], NP[typ[0]]), np.ones(7, bool), typ)
        q = O.OCol(np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1.0], NP[typ[0]]), np.ones(7, bool), typ)
        for asc, nf in ORDERS:
            keys = [(0, asc, nf)]
            bounds_check(b2, take([z], S.sort_order([z], keys)), [q], keys)


def test_search_bounds_multi_key_and_empty(b2):
    rng = np.random.default_rng(801)
    n = 4000
    cols = [few_col(rng, (O.INT32, 0, 0), n, 6, 0.1), edge_col(rng, (O.FLOAT64, 0, 0), n), few_col(rng, (O.DECIMAL128, 38, 0), n, 5, 0.1)]
    for trial in range(6):
        keys = [(k, int(rng.integers(0, 2)), int(rng.integers(0, 2))) for k in range(3)]
        sc = take(cols, S.sort_order(cols, keys))
        pc = [probe_values(rng, c, 1200) for c in cols]
        pc = [O.OCol(c.values[:1200], c.valid[:1200], c.typ) for c in pc]
        bounds_check(b2, sc, pc, keys, keys)
    empty = [O.OCol(c.values[:0], c.valid[:0], c.typ) for c in cols]
    bounds_check(b2, empty, [O.OCol(c.values[:50], c.valid[:50], c.typ) for c in cols], [(0, 1, 1), (1, 0, 0), (2, 1, 0)])
    bounds_check(b2, cols, empty, [(0, 1, 1)])


def test_search_bounds_rejects_strings_and_type_mismatches(b2):
    s = b2.Table.from_columns([b2.Column.from_strings(["a", "b"])])
    i32 = b2.Table.from_columns([b2.Column.from_numpy(np.array([1, 2], np.int32))])
    i64 = b2.Table.from_columns([b2.Column.from_numpy(np.array([1, 2], np.int64))])
    for st, pt, code in ((s, s, ERR_UNSUPPORTED), (i32, i64, ERR_INVALID), (i64, i32, ERR_INVALID)):
        with pytest.raises(b2.B2Error) as e:
            b2.search_bounds(st, pt, [(0, 1, 1)], 0)
        assert e.value.code == code


@pytest.mark.parametrize("dt", [O.DECIMAL32, O.DECIMAL64, O.DECIMAL128])
def test_search_bounds_rejects_decimal_scale_mismatch(b2, dt):
    """regression: a DECIMAL(p, 2) sorted table probed with DECIMAL(p, 4) values compared unscaled integers (1.00 sorted after
    0.5000) and returned wrong bounds without an error"""
    def dec(vals, scale):
        return b2.Table.from_columns([b2.Column.from_numpy(np.array(vals, dtype=object if dt == O.DECIMAL128 else np.int64), dtype=dt, scale=scale)])
    st = dec([100, 200, 300], 2)
    with pytest.raises(b2.B2Error) as e:
        b2.search_bounds(st, dec([5000], 4), [(0, 1, 1)], 0)
    assert e.value.code == ERR_INVALID
    assert b2.search_bounds(st, dec([150, 300], 2), [(0, 1, 1)], 1).to_pylist() == [1, 3]


# ---- operators --------------------------------------------------------------------------------------------------------------
def batches_of(rng, sizes, make):
    return [make(rng, n, b) for b, n in enumerate(sizes)]


def test_gpu_sort_exec_global_and_per_batch(b2):
    rng = np.random.default_rng(901)
    sizes = [1200, 0, 3000, 17, 900]

    def make(rng, n, b):
        return [edge_col(rng, (O.INT64, 0, 0), n), edge_col(rng, (O.STRING, 0, 0), n), edge_col(rng, (O.FLOAT32, 0, 0), n), index_col(n, b * 100000)]
    parts = batches_of(rng, sizes, make)
    keys = [(2, 0, 1), (1, 1, 0), (0, 1, 1)]
    out = E.GpuSortExec(keys, E.GpuBatchSource([table(b2, p) for p in parts]), global_sort=True).collect()
    cat = S.concat(parts)
    assert_cols(out, cat, S.sort_order(cat, keys), "global")
    outs = [t for t in E.GpuSortExec(keys, E.GpuBatchSource([table(b2, p) for p in parts]), global_sort=False) if t.num_rows]
    nonempty = [p for p in parts if len(p[0].valid)]
    assert len(outs) == len(nonempty)
    for got, p in zip(outs, nonempty):
        assert_cols(got, p, S.sort_order(p, keys), "per batch")


def test_gpu_topn_across_batches(b2):
    """GpuTopN folds per-batch top-Ns: ties across batches keep the earlier batch first; empty batches; limit 0; a limit above
    the input; one batch large enough for the radix select"""
    rng = np.random.default_rng(902)

    def make(rng, n, b):
        return [few_col(rng, (O.INT16, 0, 0), n, 6, 0.15), few_col(rng, (O.DECIMAL64, 18, 2), n, 3, 0.1), index_col(n, b * 1000000)]
    parts = batches_of(rng, [500, 0, 800, 300, 0, 1], make)
    cat = S.concat(parts)
    for keys in ([(0, 1, 1)], [(0, 0, 0)], [(1, 0, 1), (0, 1, 0)]):
        for limit in (0, 1, 7, 300, 1601, 5000):
            out = E.GpuTopN(limit, keys, E.GpuBatchSource([table(b2, p) for p in parts])).collect()
            exp = S.top_n(cat, keys, limit)
            if out is None:
                assert len(exp) == 0
            else:
                assert_cols(out, cat, exp, (keys, limit))
    big = [i64_col(rng.integers(-2**63, 2**63 - 1, TOPN_ROWS, dtype=np.int64), rng.random(TOPN_ROWS) >= 0.05), index_col(TOPN_ROWS, 5000000)]
    small = [i64_col(rng.integers(-2**63, 2**63 - 1, 2000, dtype=np.int64)), index_col(2000, 6000000)]
    small[0].values[:50] = np.sort(big[0].values)[:50]   # ties with the big batch's winners: the earlier batch comes first
    parts = [small, big, [small[0], index_col(2000, 7000000)]]
    cat = S.concat(parts)
    keys = [(0, 1, 0)]
    out, names = profiled(b2, lambda: E.GpuTopN(100, keys, E.GpuBatchSource([table(b2, p) for p in parts])).collect())
    assert TOPN_MASK in names, names
    assert_cols(out, cat, S.top_n(cat, keys, 100), "select batch")
