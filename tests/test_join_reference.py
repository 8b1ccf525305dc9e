"""The hash-join reference of test_join_paths_gpu.py (join_maps) against the oracle (oracle.spark_relational.hash_join) for
every join kind, both NULL rules and the key shapes the GPU tests use; and its restatement of the table's hash against
the CUDA sources, so that the inputs built from it (tag collisions, wrap-around chains) keep colliding when the hash
changes.  Runs without a GPU."""
import os
import re

import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_relational as R
from tests import test_join_paths_gpu as T

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark-rapids_b200", "csrc")
N = 2000


def _strings(rng, n):
    pool = np.array([b"", b"a", b"a\x00", b"\x00", b"\x00a", b"ab", b"abc", b"abcd", b"abcdefgh", b"abcdefghi", "été".encode(), b"A"], dtype=object)
    return pool[rng.integers(0, len(pool), n)]


def _floats(rng, n, npt):
    return T.float_keys(rng, n, npt)


def _cols(rng, shape, n):
    def nulls(cols):
        for c in cols:
            c.valid = rng.random(n) > 0.15
        return cols
    if shape == "i64":
        return nulls([T.ocol(rng.integers(-50, 50, n).astype(np.int64), O.INT64)])
    if shape == "i8_i16_bool":
        return nulls([T.ocol(rng.integers(-128, 128, n).astype(np.int8), O.INT8), T.ocol(rng.integers(-3, 3, n).astype(np.int16), O.INT16),
                      T.ocol(rng.integers(0, 2, n).astype(np.int8), O.BOOL8)])
    if shape == "f64":
        return nulls([T.ocol(_floats(rng, n, np.float64), O.FLOAT64)])
    if shape == "f32_i32":
        return nulls([T.ocol(_floats(rng, n, np.float32), O.FLOAT32), T.ocol(rng.integers(-2, 2, n).astype(np.int32), O.INT32)])
    if shape == "string":
        return nulls([T.ocol(_strings(rng, n), O.STRING)])
    if shape == "dec128_string":
        d = np.array([int(x) * (1 << 64) + int(y) for x, y in zip(rng.integers(-3, 3, n), rng.integers(0, 5, n))], dtype=object)
        return nulls([T.ocol(d, (O.DECIMAL128, 30, 4)), T.ocol(_strings(rng, n), O.STRING)])
    if shape == "date_dec32_ts":
        return nulls([T.ocol(rng.integers(-3, 3, n).astype(np.int32), O.DATE32), T.ocol(np.array([int(x) for x in rng.integers(-5, 5, n)], dtype=object), (O.DECIMAL32, 8, 2)),
                      T.ocol(rng.integers(-2, 2, n).astype(np.int64), O.TIMESTAMP_US)])
    raise AssertionError(shape)


SHAPES = ["i64", "i8_i16_bool", "f64", "f32_i32", "string", "dec128_string", "date_dec32_ts"]


@pytest.mark.parametrize("shape", SHAPES)
def test_reference_is_pinned_to_the_oracle(shape):
    rng = np.random.default_rng(SHAPES.index(shape))
    build, probe = _cols(rng, shape, N), _cols(rng, shape, N + 37)
    for ne in (False, True):
        maps = T.join_maps_all(build, probe, ne)
        for kind in T.KINDS:
            elm, erm = R.hash_join(build, probe, kind, ne)
            lm, rm = maps[kind]
            if rm is None:
                assert erm is None and lm.tolist() == elm, (shape, kind, ne)
            else:
                assert sorted(zip(lm.tolist(), rm.tolist())) == sorted(zip(elm, erm)), (shape, kind, ne)
            if kind == T.INNER:
                assert len(lm) > 0
        keys = [k for k in (R._join_key(build, i, ne) for i in range(N)) if k is not None]
        assert T.build_is_distinct(build, ne) == (len(set(keys)) == len(keys))


def test_reference_special_keys():
    """NaN of every bit pattern is one key, -0.0 is 0.0, an empty string is not NULL, strings differing in a trailing
    NUL byte differ, and DECIMAL128 keys differ in the high word"""
    f = np.array([T.NAN64, 0x7FF0000000000001, 0xFFF8000000000000, 0x8000000000000000, 0], dtype=np.uint64).view(np.float64)
    lm, rm = T.join_maps([T.ocol(f[:1], O.FLOAT64)], [T.ocol(f, O.FLOAT64)], T.INNER)
    assert lm.tolist() == [0, 1, 2]
    lm, rm = T.join_maps([T.ocol(f[3:4], O.FLOAT64)], [T.ocol(f, O.FLOAT64)], T.INNER)
    assert lm.tolist() == [3, 4]
    s = np.array([b"", b"a", b"a\x00"], dtype=object)
    lm, rm = T.join_maps([T.ocol(s, O.STRING)], [T.ocol(s, O.STRING, np.array([True, True, False]))], T.LEFT_OUTER)
    assert sorted(zip(lm.tolist(), rm.tolist())) == [(0, 0), (1, 1), (2, T.INT32_MIN)]
    d = np.array([[5, 1], [5, 2]], dtype=np.uint64)
    lm, rm = T.join_maps([T.ocol(d[:1], (O.DECIMAL128, 38, 0))], [T.ocol(d, (O.DECIMAL128, 38, 0))], T.SEMI)
    assert lm.tolist() == [0]


# ---- the restated hash against the sources --------------------------------------------------------------------------
def _code(name):
    with open(os.path.join(CSRC, name)) as fh:
        text = fh.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"\s+", " ", re.sub(r"//[^\n]*", "", text))


# each restated piece of test_join_paths_gpu.py and the source text it restates
RESTATED = {
    "rowops.cuh": [
        ("mix64 / MIX_M1 / MIX_M2", "x ^= x >> 33; x *= 0x%xull; x ^= x >> 33; x *= 0x%xull; x ^= x >> 33; return x;" % (T.MIX_M1, T.MIX_M2)),
        ("key_bits: float32 NaN / zero", "if (f != f) return 0x7fc00000u; if (f == 0.0f) return 0; return __float_as_uint(f);"),
        ("key_bits: float64 NaN / zero", "if (d != d) return 0x%016xull; if (d == 0.0) return 0;" % T.NAN64),
        ("key_bits: zero extension", "case 1: return reinterpret_cast<const uint8_t*>(k.data)[r]; case 2: return reinterpret_cast<const uint16_t*>(k.data)[r]; "
                                     "case 4: return reinterpret_cast<const uint32_t*>(k.data)[r]; default: return reinterpret_cast<const uint64_t*>(k.data)[r];"),
        ("row_hash: seed GOLDEN", "uint64_t h = 0x%xull;" % T.GOLDEN),
        ("row_hash: NULL_SALT", "if (!row_valid(k.valid, r)) { h = mix64(h ^ 0x%xu); continue; }" % T.NULL_SALT),
        ("row_hash: FNV_BASIS / FNV_PRIME", "uint64_t s = 0x%xull; for (int32_t q = b; q < e; q++) { s ^= p[q]; s *= 0x%xull; } h = mix64(h ^ s ^ (uint64_t)(e - b));"
         % (T.FNV_BASIS, T.FNV_PRIME)),
        ("row_hash: DECIMAL128 words", "h = mix64(h ^ p[0]); h = mix64(h ^ p[1]);"),
        ("row_hash: fixed width", "h = mix64(h ^ key_bits(k, r));"),
        ("fold32", "return (uint32_t)(h ^ (h >> 32));"),
    ],
    "join.cu": [
        ("hash_packed: packing", "bits |= key_bits(ks.c[i], r) << shift; shift += 8 * ks.c[i].width;"),
        ("hash_packed", "const uint64_t h = mix64(kb ^ 0x%xull); return (uint32_t)(h ^ (h >> 32));" % T.GOLDEN),
        ("the one-key probe packs like pack_join_key", "const uint64_t kb = (uint64_t)(UK)keys[src]; const uint32_t hh = hash_packed(kb); uint32_t idx = hh & mask;"),
        ("start slot = tag & mask", "uint32_t idx = h & mask;"),
        ("capacity", "int64_t cap = 1024; while (cap < t->rows * 2) cap <<= 1;"),
        ("layout rule", "jt->fast = fixed && kw <= 8 && !(jt->nulls_equal && nullable);"),
        ("Bloom threshold BLOOM_ROWS", "if (t->rows >= (1 << 18) && !getenv(\"B2_JOIN_NO_BLOOM\"))"),
    ],
}


@pytest.mark.parametrize("name", sorted(RESTATED))
def test_hash_restatement_matches_the_sources(name):
    code = _code(name)
    for what, text in RESTATED[name]:
        assert re.sub(r"\s+", " ", text) in code, "%s changed: update %s in tests/test_join_paths_gpu.py" % (name, what)
    assert T.BLOOM_ROWS == 1 << 18


def _mix64_int(x):
    m = (1 << 64) - 1
    x ^= x >> 33
    x = (x * T.MIX_M1) & m
    x ^= x >> 33
    x = (x * T.MIX_M2) & m
    return x ^ (x >> 33)


def test_restated_hash_wraps_like_uint64():
    """the numpy restatement (uint64 arithmetic that wraps) against python integers reduced mod 2^64"""
    rng = np.random.default_rng(1)
    x = rng.integers(-2**63, 2**63 - 1, 1000, dtype=np.int64)
    m = (1 << 64) - 1
    want = []
    for v in x.tolist():
        h = _mix64_int((v & m) ^ T.GOLDEN)
        want.append((h ^ (h >> 32)) & 0xFFFFFFFF)
    assert T.hash_packed([(x, O.INT64)]).tolist() == want
    y = rng.integers(-2**31, 2**31, 1000).astype(np.int32)
    got = T.row_hash([("fixed", x, O.INT64), ("null", 1000), ("fixed", y, O.INT32)]).tolist()
    for i, (a, b) in enumerate(zip(x.tolist(), y.tolist())):
        h = _mix64_int(_mix64_int(_mix64_int(T.GOLDEN ^ (a & m)) ^ T.NULL_SALT) ^ (b & 0xFFFFFFFF))
        assert got[i] == (h ^ (h >> 32)) & 0xFFFFFFFF
    raw = rng.integers(0, 256, (50, 8), dtype=np.uint8)
    got = T.row_hash([("string", raw)]).tolist()
    for i, r in enumerate(raw):
        s = T.FNV_BASIS
        for byte in r.tolist():
            s = ((s ^ byte) * T.FNV_PRIME) & m
        h = _mix64_int(T.GOLDEN ^ s ^ 8)
        assert got[i] == (h ^ (h >> 32)) & 0xFFFFFFFF
    i, j = T.tag_collisions(T.hash_packed([(np.unique(rng.integers(-2**63, 2**63 - 1, 1 << 20, dtype=np.int64)), O.INT64)]))
    assert len(i) >= 50 and (i != j).all()
