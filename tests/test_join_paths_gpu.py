"""Every build and probe path of the hash join (join.cu) against an exact reference, at the inputs where a hash table goes
wrong: keys that share a 32-bit tag, probe chains that wrap past the end of the table, long chains, NaN / -0.0 keys,
NULL keys with bytes under them that equal a build key, narrow packed keys of negative values, outputs past 2^31 - 1
rows.  The paths and how the inputs reach them (the rules of b2_join_build / b2_join_probe_sel):
 * packed table     every build key fixed width (not STRING / DECIMAL128), <= 8 bytes together, and not (nulls_equal
                    with a build key column that has a validity buffer): 16-byte slots {tag | row, packed key}
 * generic table    otherwise: 8-byte slots, keys compared by rows_equal
 * distinct         no two build rows share a key: INNER / LEFT OUTER (and FULL OUTER's left outer part) take the
                    single-pass probes; a build side with duplicates, and every SEMI / ANTI, take count + write
 * distinct1        INNER, distinct, packed, one key of width 4 or 8, not a float, probe key column without a validity
                    buffer: join_probe_distinct1_kernel
 * Bloom filter     build rows >= 2^18 (B2_JOIN_NO_BLOOM unset)
Each probe asserts from the kernel timings which probe kernel ran.  The table layout and the Bloom filter are not
visible from outside, so the inputs reach them by construction.  The tag and start slot of a key are computed by a numpy
restatement of the table's hash (mix64 / hash_packed / row_hash), which test_join_reference.py pins to the sources."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import spark_cpu as O

pytestmark = pytest.mark.gpu

INT32_MIN = -2**31
INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER = range(5)
KINDS = [INNER, LEFT_OUTER, SEMI, ANTI, FULL_OUTER]
PROBE_KERNELS = {"join_probe_distinct1_kernel", "join_probe_distinct_kernel", "join_probe_count_kernel", "join_probe_write_kernel",
                 "join_filter_probe_kernel"}
BLOOM_ROWS = 1 << 18
ERR_INVALID, ERR_SIZE_OVERFLOW = 1, 4
_WIDTH = {O.BOOL8: 1, O.INT8: 1, O.INT16: 2, O.INT32: 4, O.INT64: 8, O.FLOAT32: 4, O.FLOAT64: 8, O.DATE32: 4, O.TIMESTAMP_US: 8,
          O.DECIMAL32: 4, O.DECIMAL64: 8, O.DECIMAL128: 16}
_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
_SIGNED = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}
NAN64 = 0x7FF8000000000000


# ---- the exact reference -----------------------------------------------------------------------------------------
def _float_words(values):
    """Spark's normalised join key: every NaN one value, -0.0 == 0.0; then the bits (float32 widens exactly)"""
    with np.errstate(invalid="ignore"):
        f = np.asarray(values, dtype=np.float64).copy()
    f[f == 0] = 0.0
    bits = f.view(np.int64).copy()
    bits[np.isnan(f)] = NAN64
    return bits


def _dec128_words(values):
    """(n, 2) uint64 words, or python ints -> (lo, hi) int64"""
    v = np.asarray(values)
    if v.ndim == 2:
        w = np.ascontiguousarray(v, dtype=np.uint64).view(np.int64)
        return [w[:, 0].copy(), w[:, 1].copy()]
    m = (1 << 64) - 1
    lo = np.array([((int(x) & m) ^ (1 << 63)) - (1 << 63) for x in v], dtype=np.int64)
    hi = np.array([int(x) >> 64 for x in v], dtype=np.int64)
    return [lo, hi]


def _words(c):
    dt = c.typ[0]
    if dt in (O.FLOAT32, O.FLOAT64):
        return [_float_words(c.values)]
    if dt == O.DECIMAL128:
        return _dec128_words(c.values)
    if dt == O.BOOL8:
        return [(np.asarray(c.values) != 0).astype(np.int64)]
    return [np.asarray(c.values).astype(np.int64)]


def _row_ids(build, probe):
    """one int64 id per row of build and of probe: equal ids = equal keys (NULL equal to NULL); and the any-NULL flags"""
    nb, npr = len(build[0]), len(probe[0])
    cols, nulls = [], np.zeros(nb + npr, bool)
    for bc, pc in zip(build, probe):
        valid = np.concatenate([bc.valid, pc.valid])
        if bc.typ[0] == O.STRING:
            both = np.empty(nb + npr, dtype=object)
            both[:nb], both[nb:] = bc.values, pc.values
            ws = [np.unique(both, return_inverse=True)[1].reshape(-1).astype(np.int64)] if nb + npr else [np.zeros(0, np.int64)]
        else:
            ws = [np.concatenate([a, b]) for a, b in zip(_words(bc), _words(pc))]
        cols += [np.where(valid, w, 0) for w in ws]
        if not valid.all():
            cols.append((~valid).astype(np.int64))
        nulls |= ~valid
    if len(cols) == 1 or nb + npr == 0:
        ids = cols[0]
    else:
        ids = np.unique(np.stack(cols, axis=1), axis=0, return_inverse=True)[1].reshape(-1)
    return ids[:nb], ids[nb:], nulls[:nb], nulls[nb:]


def join_maps_all(build_cols, probe_cols, nulls_equal, kinds=KINDS):
    """{kind: (left map, right map | None)} as int64 arrays; stream = probe = left.  With nulls_equal false a row with any
    NULL key matches nothing.  INNER / LEFT OUTER pairs come in stream order, LEFT OUTER adds (r, INT32_MIN) for unmatched
    stream rows, SEMI / ANTI give stream rows in stream order, FULL OUTER adds (INT32_MIN, b) for unmatched build rows."""
    bid, pid, bnull, pnull = _row_ids(build_cols, probe_cols)
    nb, npr = len(bid), len(pid)
    bi = np.arange(nb) if nulls_equal else np.flatnonzero(~bnull)
    order = bi[np.argsort(bid[bi], kind="stable")]
    bs = bid[order]
    rows = np.arange(npr) if nulls_equal else np.flatnonzero(~pnull)
    lo, hi = np.searchsorted(bs, pid[rows], "left"), np.searchsorted(bs, pid[rows], "right")
    cnt_rows = hi - lo
    cnt = np.zeros(npr, np.int64)
    cnt[rows] = cnt_rows
    left = np.repeat(rows, cnt_rows).astype(np.int64)
    start = np.repeat(lo - (np.cumsum(cnt_rows) - cnt_rows), cnt_rows)
    right = order[start + np.arange(len(left))].astype(np.int64) if len(left) else np.zeros(0, np.int64)
    out = {}
    lonely = np.flatnonzero(cnt == 0)
    lo_l = np.concatenate([left, lonely])
    lo_r = np.concatenate([right, np.full(len(lonely), INT32_MIN, np.int64)])
    for kind in kinds:
        if kind == INNER:
            out[kind] = (left, right)
        elif kind == LEFT_OUTER:
            out[kind] = (lo_l, lo_r)
        elif kind == SEMI:
            out[kind] = (np.flatnonzero(cnt > 0).astype(np.int64), None)
        elif kind == ANTI:
            out[kind] = (lonely.astype(np.int64), None)
        else:
            hit = np.zeros(nb, bool)
            hit[right] = True
            unb = np.flatnonzero(~hit)
            out[kind] = (np.concatenate([lo_l, np.full(len(unb), INT32_MIN, np.int64)]), np.concatenate([lo_r, unb]))
    return out


def join_maps(build_cols, probe_cols, kind, nulls_equal=False):
    return join_maps_all(build_cols, probe_cols, nulls_equal, [kind])[kind]


def build_is_distinct(build_cols, nulls_equal):
    bid, _, bnull, _ = _row_ids(build_cols, [O.OCol(c.values[:0], c.valid[:0], c.typ) for c in build_cols])
    live = bid if nulls_equal else bid[~bnull]
    return len(np.unique(live)) == len(live)


# ---- the table's hash, restated (pinned to rowops.cuh / join.cu by test_join_reference.py) --------------------------
U64 = np.uint64
GOLDEN, NULL_SALT, FNV_BASIS, FNV_PRIME = 0x9E3779B97F4A7C15, 0x5BD1E995, 0xCBF29CE484222325, 0x100000001B3
MIX_M1, MIX_M2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53


def mix64(x):
    x = x ^ (x >> U64(33))
    x = x * U64(MIX_M1)
    x = x ^ (x >> U64(33))
    x = x * U64(MIX_M2)
    return x ^ (x >> U64(33))


def fold32(h):
    return (h ^ (h >> U64(32))) & U64(0xFFFFFFFF)


def key_bits(values, dtype):
    """key_bits: the value's bytes zero-extended (floats normalised)"""
    if dtype in (O.FLOAT32, O.FLOAT64):
        f = np.asarray(values, dtype=np.float32 if dtype == O.FLOAT32 else np.float64).copy()
        w = _WIDTH[dtype]
        f[f == 0] = 0
        bits = f.view(_UNSIGNED[w]).astype(U64)
        bits[np.isnan(f)] = 0x7FC00000 if w == 4 else NAN64
        return bits
    w = _WIDTH[dtype]
    return np.asarray(values).astype(_SIGNED[w]).view(_UNSIGNED[w]).astype(U64)


def hash_packed(cols):
    """tag of a packed key: cols = [(values, dtype)], packed low column first"""
    kb, shift = np.zeros(len(cols[0][0]), U64), 0
    for v, dt in cols:
        kb = kb | (key_bits(v, dt) << U64(shift))
        shift += 8 * _WIDTH[dt]
    return fold32(mix64(kb ^ U64(GOLDEN)))


def row_hash(cols):
    """tag of a generic key: cols = [("fixed", values, dtype) | ("string", (n, L) uint8 bytes) | ("dec128", (n, 2) uint64)
    | ("null", n)]"""
    n = cols[0][1] if cols[0][0] == "null" else len(cols[0][1])
    h = np.full(n, GOLDEN, U64)
    for c in cols:
        if c[0] == "null":
            h = mix64(h ^ U64(NULL_SALT))
        elif c[0] == "string":
            b = np.asarray(c[1], np.uint8)
            s = np.full(n, FNV_BASIS, U64)
            for q in range(b.shape[1]):
                s = (s ^ b[:, q].astype(U64)) * U64(FNV_PRIME)
            h = mix64(h ^ s ^ U64(b.shape[1]))
        elif c[0] == "dec128":
            w = np.asarray(c[1], U64)
            h = mix64(mix64(h ^ w[:, 0]) ^ w[:, 1])
        else:
            h = mix64(h ^ key_bits(c[1], c[2]))
    return fold32(h)


def capacity(build_rows):
    cap = 1024
    while cap < 2 * build_rows:
        cap <<= 1
    return cap


def tag_collisions(tags):
    """index pairs (i, j), i != j, of equal tags (each tag once)"""
    o = np.argsort(tags, kind="stable")
    st = tags[o]
    k = np.flatnonzero(st[1:] == st[:-1])
    k = k[np.r_[True, st[k[1:]] != st[k[:-1]]]] if len(k) else k
    return o[k], o[k + 1]


# ---- running a probe -----------------------------------------------------------------------------------------------
def key_of(ids):
    """distinct int64 keys, both signs, spread over all 64 bits (an odd multiplier is a bijection)"""
    with np.errstate(over="ignore"):
        return (np.asarray(ids).astype(np.int64) * np.int64(-7046029254386353131)) ^ np.int64(0x5DEECE66D)


def ocol(values, typ, valid=None):
    n = len(values)
    return O.OCol(values, np.ones(n, bool) if valid is None else valid, typ if isinstance(typ, tuple) else (typ, 0, 0))


def to_column(b2, c, force_validity=False):
    dt, _, scale = c.typ
    valid = c.valid if (force_validity or not c.valid.all()) else None
    if dt == O.STRING:
        vals = list(c.values)
        lens = np.array([len(v) for v in vals], dtype=np.int64)
        offs = np.zeros(len(vals) + 1, np.int32)
        offs[1:] = np.cumsum(lens)
        chars = np.frombuffer(b"".join(vals), dtype=np.uint8) if len(vals) else np.zeros(0, np.uint8)
        return b2.Column.from_string_buffers(chars, offs, valid=valid)
    if dt == O.DECIMAL128:
        v = np.asarray(c.values)
        return b2.Column.from_numpy(v if v.ndim == 2 else np.array([int(x) for x in v], dtype=object), dtype=dt, valid=valid, scale=scale)
    if dt in (O.DECIMAL32, O.DECIMAL64):
        return b2.Column.from_numpy(np.asarray(c.values).astype(np.int64), dtype=dt, valid=valid, scale=scale)
    return b2.Column.from_numpy(np.asarray(c.values), dtype=dt, valid=valid, scale=scale)


def to_table(b2, cols, force_validity=False):
    return b2.Table.from_columns([to_column(b2, c, force_validity) for c in cols])


def is_packed(build_cols, nulls_equal):
    fixed = all(c.typ[0] not in (O.STRING, O.DECIMAL128) for c in build_cols)
    width = sum(_WIDTH.get(c.typ[0], 0) for c in build_cols)
    has_buffer = any(not c.valid.all() for c in build_cols)
    return fixed and width <= 8 and not (nulls_equal and has_buffer)


def expected_kernels(build_cols, probe_cols, kind, nulls_equal, n, total, probe_buffer=None):
    """the probe kernels b2_join_probe_sel launches for n probe rows and `total` output rows"""
    if n == 0:
        return set()
    distinct = build_is_distinct(build_cols, nulls_equal)
    if distinct and kind in (INNER, LEFT_OUTER, FULL_OUTER):
        p = probe_cols[0]
        buf = (not p.valid.all()) if probe_buffer is None else probe_buffer
        if (kind == INNER and is_packed(build_cols, nulls_equal) and len(build_cols) == 1 and p.typ[0] not in (O.FLOAT32, O.FLOAT64)
                and _WIDTH[p.typ[0]] in (4, 8) and not buf):
            return {"join_probe_distinct1_kernel"}
        return {"join_probe_distinct_kernel"}
    if kind == FULL_OUTER:
        total = n
    return {"join_probe_count_kernel"} | ({"join_probe_write_kernel"} if total else set())


def probe(b2, ht, probe_table, kind, selection=None):
    """-> (left map, right map | None) as int64 arrays, the probe kernels that ran"""
    b2.profile_enable(True)
    try:
        lm, rm = ht.probe(probe_table, kind, selection=selection)
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return (lm.to_numpy()[0].astype(np.int64), None if rm is None else rm.to_numpy()[0].astype(np.int64)), names & PROBE_KERNELS


def sorted_pairs(lm, rm):
    o = np.lexsort((rm, lm))
    return lm[o], rm[o]


def assert_maps(kind, got, want, what=""):
    (gl, gr), (wl, wr) = got, want
    if kind in (SEMI, ANTI):
        assert gr is None, what
        assert np.array_equal(gl, wl), (what, len(gl), len(wl))
    else:
        assert len(gl) == len(wl), (what, len(gl), len(wl))
        a, b = sorted_pairs(gl, gr), sorted_pairs(wl, wr)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), what


def check_join(b2, build, probe_cols, kinds=KINDS, nulls_equal=(False, True), what=""):
    """every kind x nulls_equal: maps against the reference and the probe kernel against the rules"""
    pt = to_table(b2, probe_cols)
    for ne in nulls_equal:
        ht = b2.JoinHashTable(to_table(b2, build), ne)
        want = join_maps_all(build, probe_cols, ne, kinds)
        for kind in kinds:
            got, ran = probe(b2, ht, pt, kind)
            tag = (what, kind, ne)
            assert_maps(kind, got, want[kind], tag)
            assert ran == expected_kernels(build, probe_cols, kind, ne, len(probe_cols[0]), len(want[kind][0])), (tag, ran)


# ---- 2. the path matrix ----------------------------------------------------------------------------------------------
NPROBE = 300_000


def matrix_keys(layout, ids):
    if layout == "packed":                     # one INT64 key: packed, and the one-key distinct probe for INNER
        return [ocol(key_of(ids), O.INT64)]
    return [ocol(key_of(ids), O.INT64), ocol((ids % 2001 - 1000).astype(np.int32), O.INT32)]   # 12 bytes: generic


def matrix_input(layout, dup, nb, seed):
    rng = np.random.default_rng(seed)
    if dup:                                    # every key twice (one three times when nb is odd)
        ids = np.resize(rng.permutation(2 * nb)[: (nb + 1) // 2], nb)
        rng.shuffle(ids)
    else:
        ids = rng.permutation(4 * nb)[:nb]
    pids = np.where(rng.random(NPROBE) < 0.5, rng.choice(ids, NPROBE), 4 * nb + rng.integers(0, 4 * nb, NPROBE))   # half absent
    return matrix_keys(layout, ids), matrix_keys(layout, pids)


def selections(rng, n):
    sparse = np.flatnonzero(rng.random(n) < 0.15)
    sparse = np.unique(np.r_[sparse, n - 1]).astype(np.int32)
    return {"none": None, "empty": np.zeros(0, np.int32), "all": np.arange(n, dtype=np.int32), "sparse": sparse}


def take(cols, idx):
    return [O.OCol(c.values[idx], c.valid[idx], c.typ) for c in cols]


@pytest.mark.parametrize("nb", [100_000, BLOOM_ROWS, BLOOM_ROWS + 1], ids=["bloom_off", "bloom_2^18", "bloom_2^18+1"])
@pytest.mark.parametrize("dup", [False, True], ids=["distinct", "duplicates"])
@pytest.mark.parametrize("layout", ["packed", "generic"])
def test_path_matrix(b2, monkeypatch, layout, dup, nb):
    """kinds 0-4 on one table, through no selection vector, an empty one, one of every row and a sparse one ending at the
    last row (never FULL OUTER); with the Bloom filter on, the same maps with B2_JOIN_NO_BLOOM=1"""
    monkeypatch.delenv("B2_JOIN_NO_BLOOM", raising=False)
    monkeypatch.delenv("B2_JOIN_NO_FAST_PROBE", raising=False)
    build, pr = matrix_input(layout, dup, nb, seed=nb + 7 * dup + (layout == "generic"))
    assert build_is_distinct(build, False) == (not dup)
    ht = b2.JoinHashTable(to_table(b2, build))
    pt = to_table(b2, pr)
    rng = np.random.default_rng(11)
    for sname, sel in selections(rng, NPROBE).items():
        sub = pr if sel is None else take(pr, sel)
        want = join_maps_all(build, sub, False)
        for kind in KINDS:
            if kind == FULL_OUTER and sel is not None:
                continue
            got, ran = probe(b2, ht, pt, kind, None if sel is None else b2.Column.from_numpy(sel))
            w = want[kind]
            if sel is not None:                 # the left map carries original row ids
                w = (sel.astype(np.int64)[w[0]], w[1])
            assert_maps(kind, got, w, (sname, kind))
            assert ran == expected_kernels(build, sub, kind, False, len(sub[0]), len(w[0])), (sname, kind, ran)
            if kind == INNER and sel is None:
                assert 0.3 * NPROBE < len(got[0]) < 1.5 * NPROBE        # about half the probe rows match
    with pytest.raises(b2.B2Error) as e:
        ht.probe(pt, FULL_OUTER, selection=b2.Column.from_numpy(np.arange(5, dtype=np.int32)))
    assert e.value.code == ERR_INVALID
    if nb >= BLOOM_ROWS:
        monkeypatch.setenv("B2_JOIN_NO_BLOOM", "1")
        ht2 = b2.JoinHashTable(to_table(b2, build))
        for kind in KINDS:
            a, _ = probe(b2, ht, pt, kind)
            b, _ = probe(b2, ht2, pt, kind)
            assert_maps(kind, a, b, ("bloom vs no bloom", kind))


@pytest.mark.parametrize("nb", [100_000, BLOOM_ROWS], ids=["bloom_off", "bloom_on"])
def test_probe_kernels_agree(b2, monkeypatch, nb):
    """INNER against a distinct packed table: join_probe_distinct1_kernel, the generic single-pass kernel under
    B2_JOIN_NO_FAST_PROBE=1, and the generic kernel again for a probe key column with a validity buffer and no NULL"""
    monkeypatch.delenv("B2_JOIN_NO_FAST_PROBE", raising=False)
    for kt in (np.int64, np.int32):
        build, pr = matrix_input("packed", False, nb, seed=3)
        build = [ocol(build[0].values.astype(kt), O.INT64 if kt == np.int64 else O.INT32)]
        pr = [ocol(pr[0].values.astype(kt), build[0].typ)]
        ht = b2.JoinHashTable(to_table(b2, build))
        want = join_maps(build, pr, INNER)
        fast, ran = probe(b2, ht, to_table(b2, pr), INNER)
        assert ran == {"join_probe_distinct1_kernel"}, ran
        buffered, ran = probe(b2, ht, to_table(b2, pr, force_validity=True), INNER)
        assert ran == {"join_probe_distinct_kernel"}, ran
        monkeypatch.setenv("B2_JOIN_NO_FAST_PROBE", "1")
        slow, ran = probe(b2, ht, to_table(b2, pr), INNER)
        monkeypatch.delenv("B2_JOIN_NO_FAST_PROBE")
        assert ran == {"join_probe_distinct_kernel"}, ran
        for got in (fast, buffered, slow):
            assert_maps(INNER, got, want, kt)


BLOOM_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import spark_rapids_b200 as b2
b2.init(0)
n = 1 << 18
key_of = lambda ids: (ids.astype(np.int64) * np.int64(-7046029254386353131)) ^ np.int64(0x5DEECE66D)
keys = key_of(np.arange(n))
absent = key_of(np.arange(n, n + 100_000))
ht = b2.JoinHashTable(b2.Table.from_columns([b2.Column.from_numpy(keys)]))
probe = np.concatenate([keys[::-1], absent])
lm, rm = ht.probe(b2.Table.from_columns([b2.Column.from_numpy(probe)]), b2.JOIN_INNER)
l, r = lm.to_numpy()[0], rm.to_numpy()[0]
o = np.argsort(r)
assert len(r) == n and np.array_equal(r[o], np.arange(n)) and np.array_equal(l[o], n - 1 - np.arange(n)), len(r)
semi, _ = ht.probe(b2.Table.from_columns([b2.Column.from_numpy(probe)]), b2.JOIN_LEFT_SEMI)
assert np.array_equal(semi.to_numpy()[0], np.arange(n)), len(semi)
print("every build key found")
"""


@pytest.mark.parametrize("env", [{"B2_JOIN_BLOOM_K": "2"}, {"B2_JOIN_BLOOM_K": "4", "B2_JOIN_BLOOM_BITS": "16"}], ids=["k2", "k4_bits16"])
def test_bloom_settings_in_a_child_process(env):
    """the Bloom settings are read once per process: a child builds a 2^18-row table with k = 2 (k = 4 sets the third and
    fourth bit of bloom_of) and finds every build key, through the one-key probe and the count / write probe"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    e = dict(os.environ)
    e.pop("B2_JOIN_NO_BLOOM", None)
    e.update(env)
    p = subprocess.run([sys.executable, "-c", BLOOM_CHILD, root], cwd=root, env=e, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "every build key found" in p.stdout, p.stdout + p.stderr


# ---- 3. key types and shapes ---------------------------------------------------------------------------------------
FLOAT_SPECIALS = np.array([NAN64, 0x7FF0000000000001, 0xFFF8000000000000, 0x8000000000000000, 0, 0x7FF0000000000000,
                           0xFFF0000000000000], dtype=np.uint64).view(np.float64)   # NaNs, -0.0, 0.0, +inf, -inf


@np.errstate(invalid="ignore")                        # NaN payloads narrowed to float32
def float_keys(rng, n, npt):
    v = np.round(rng.standard_normal(n) * 20).astype(npt) / npt(4)
    special = rng.random(n) < 0.3
    s = FLOAT_SPECIALS[rng.integers(0, len(FLOAT_SPECIALS), n)].astype(npt)
    if npt == np.float32:                      # float32 NaNs with their own bit patterns
        nan32 = np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0x7FFFFFFF], np.uint32).view(np.float32)
        isn = np.isnan(s)
        s[isn] = nan32[rng.integers(0, 4, int(isn.sum()))]
    return np.where(special, s, v).astype(npt)


@pytest.mark.parametrize("shape", ["f64_packed", "f64_i64_generic", "f32_i32_packed"])
def test_float_keys(b2, shape):
    """NaN of several bit patterns matches NaN, -0.0 matches 0.0, +-inf match themselves, on both sides"""
    rng = np.random.default_rng(len(shape))
    for nb, npr in ((400, 3000), (3000, 3000)):
        def keys(n):
            if shape == "f64_packed":
                return [ocol(float_keys(rng, n, np.float64), O.FLOAT64)]
            if shape == "f64_i64_generic":
                return [ocol(float_keys(rng, n, np.float64), O.FLOAT64), ocol(rng.integers(-2, 2, n).astype(np.int64), O.INT64)]
            return [ocol(float_keys(rng, n, np.float32), O.FLOAT32), ocol(rng.integers(-2, 2, n).astype(np.int32), O.INT32)]
        build, pr = keys(nb), keys(npr)
        if nb == 400:                          # a distinct build side: one row per normalised key
            bid = _row_ids(build, build)[0]
            first = np.unique(bid, return_index=True)[1]
            build = take(build, np.sort(first))
        assert is_packed(build, False) == shape.endswith("packed")
        want = join_maps(build, pr, INNER)
        bk = _float_words(build[0].values)
        pk = _float_words(pr[0].values[want[0]])
        assert np.array_equal(bk[want[1]], pk)
        isn = np.isnan(pr[0].values[want[0]].astype(np.float64))
        assert isn.any() and (pr[0].values[want[0]] == 0).any()          # NaN and zero keys do match
        assert len(np.unique(pr[0].values[want[0]][isn].astype(np.float64).view(np.uint64))) >= 2 or shape.startswith("f32")
        check_join(b2, build, pr, what=(shape, nb))


def _neg_ints(rng, n, npt, k):
    """values of both signs, k distinct"""
    info = np.iinfo(npt)
    prng = np.random.default_rng(k)                      # the same pool on both sides
    pool = np.unique(np.r_[np.array([info.min, -1, 0, 1, info.max], npt), prng.integers(info.min, info.max, 4 * k, dtype=np.int64).astype(npt)])
    pool = np.r_[pool[pool < 0][: k // 2], pool[pool >= 0][: k - k // 2]]
    return rng.choice(pool, n).astype(npt)


def shape_keys(b2, rng, shape, n):
    I = lambda npt, dt, k: ocol(_neg_ints(rng, n, npt, k), dt)                                         # noqa: E731
    if shape == "i8_i8":
        return [I(np.int8, O.INT8, 40), I(np.int8, O.INT8, 40)]
    if shape == "i16_i8_bool":
        return [I(np.int16, O.INT16, 60), I(np.int8, O.INT8, 20), ocol(rng.integers(0, 2, n).astype(np.int8), O.BOOL8)]
    if shape == "i32_i16_i8_bool":
        return [I(np.int32, O.INT32, 50), I(np.int16, O.INT16, 10), I(np.int8, O.INT8, 5), ocol(rng.integers(0, 2, n).astype(np.int8), O.BOOL8)]
    if shape == "date_i32":
        return [ocol(rng.integers(-30, 30, n).astype(np.int32) * 97, O.DATE32), I(np.int32, O.INT32, 30)]
    if shape == "dec32_i32":
        return [ocol(rng.integers(-20, 20, n).astype(np.int64) * 4_999_999, (O.DECIMAL32, 8, 2)), I(np.int32, O.INT32, 30)]
    if shape == "i64_i8":
        return [I(np.int64, O.INT64, 100), I(np.int8, O.INT8, 10)]
    if shape == "dec128_string":
        hi = rng.integers(-3, 3, n).astype(np.int64)
        d = np.stack([rng.integers(0, 40, n).astype(np.uint64), hi.view(np.uint64)], axis=1)     # negative values: hi < 0
        strs = np.array([b"", b"a", b"a\x00", b"\x00", b"ab", b"abc", b"abcdefghij", b"abcdefghijk", "été".encode()], dtype=object)
        return [ocol(d, (O.DECIMAL128, 30, 4)), ocol(strs[rng.integers(0, len(strs), n)], O.STRING)]
    if shape == "eight_keys":
        return [I(np.int8, O.INT8, 3), I(np.int16, O.INT16, 3), I(np.int32, O.INT32, 3), I(np.int64, O.INT64, 3),
                ocol(rng.integers(0, 2, n).astype(np.int8), O.BOOL8), ocol(rng.integers(-2, 2, n).astype(np.int32), O.DATE32),
                ocol(rng.integers(-2, 2, n).astype(np.int64), O.TIMESTAMP_US), ocol(rng.integers(-2, 2, n).astype(np.int64), (O.DECIMAL64, 12, 2))]
    raise AssertionError(shape)


SHAPES = ["i8_i8", "i16_i8_bool", "i32_i16_i8_bool", "date_i32", "dec32_i32", "i64_i8", "dec128_string", "eight_keys"]
PACKED_SHAPES = {"i8_i8", "i16_i8_bool", "i32_i16_i8_bool", "date_i32", "dec32_i32"}


@pytest.mark.parametrize("shape", SHAPES, ids=[s + ("-packed" if s in PACKED_SHAPES else "-generic") for s in SHAPES])
def test_key_shapes(b2, shape):
    """packed shapes of 2, 4 and 8 bytes with negative values in every column (the packing zero-extends), generic shapes
    on both sides of the 8-byte line; a distinct and a duplicate build side, no NULLs, then NULLs in every key column"""
    rng = np.random.default_rng(SHAPES.index(shape))
    for null_frac in (0.0, 0.15):
        build, pr = shape_keys(b2, rng, shape, 2500), shape_keys(b2, rng, shape, 4000)
        for c in build + pr:
            c.valid = rng.random(len(c)) >= null_frac
        assert is_packed(build, False) == (shape in PACKED_SHAPES)
        check_join(b2, build, pr, what=(shape, null_frac, "dup"))
        bid = _row_ids(build, build)[0]
        first = np.sort(np.unique(bid, return_index=True)[1])
        check_join(b2, take(build, first), pr, what=(shape, null_frac, "distinct"))


def test_key_count_and_dtype_rejected(b2):
    rng = np.random.default_rng(2)
    nine = [ocol(rng.integers(0, 3, 10).astype(np.int8), O.INT8) for _ in range(9)]
    with pytest.raises(b2.B2Error) as e:
        b2.JoinHashTable(to_table(b2, nine))
    assert e.value.code == ERR_INVALID
    ht = b2.JoinHashTable(to_table(b2, [ocol(np.arange(10, dtype=np.int32), O.INT32)]))
    for bad in ([ocol(np.arange(10, dtype=np.int64), O.INT64)], [ocol(np.arange(10, dtype=np.int32), O.DATE32)],
                [ocol(np.arange(10, dtype=np.int32), O.INT32), ocol(np.arange(10, dtype=np.int32), O.INT32)]):
        for kind in KINDS:
            with pytest.raises(b2.B2Error) as e:
                ht.probe(to_table(b2, bad), kind)
            assert e.value.code == ERR_INVALID


def test_null_keys(b2):
    """a build side whose keys are all NULL; a NULL-free build side probed with NULL keys whose bytes equal a build key
    (packed under nulls_equal, and distinct: the single-pass probe must not read the bytes of a NULL key)"""
    rng = np.random.default_rng(9)
    allnull = [ocol(rng.integers(0, 5, 300).astype(np.int64), O.INT64, np.zeros(300, bool))]
    pr = [ocol(rng.integers(0, 5, 2000).astype(np.int64), O.INT64, rng.random(2000) > 0.3)]
    check_join(b2, allnull, pr, what="all NULL build")
    for kt, dt in ((np.int64, O.INT64), (np.int32, O.INT32), (np.int16, O.INT16)):
        for dup in (False, True):
            bk = rng.permutation(5000)[:1000].astype(kt)
            if dup:
                bk = np.repeat(bk[:500], 2)
            build = [ocol(bk, dt)]
            pv = rng.choice(bk, 6000)
            valid = rng.random(6000) > 0.3
            pr = [ocol(np.where(valid, pv, bk[0]).astype(kt), dt, valid)]          # the bytes under a NULL: a build key
            check_join(b2, build, pr, what=("NULL probe", dt, dup))
        two = [ocol(rng.permutation(3000)[:800].astype(np.int32), O.INT32), ocol(rng.integers(-5, 5, 800).astype(np.int32), O.INT32)]
        pr2 = take(two, rng.integers(0, 800, 3000))
        for c in pr2:
            c.valid = rng.random(3000) > 0.25
        check_join(b2, two, pr2, what="NULL probe, two keys")


@pytest.mark.parametrize("npr", [0, 1, 31, 32, 33])
@pytest.mark.parametrize("nb", [0, 1, 31, 32, 33])
def test_sizes(b2, nb, npr):
    rng = np.random.default_rng(nb * 100 + npr)
    for cols in ((O.INT64,), (O.STRING,)):
        def keys(n):
            v = rng.integers(0, 20, n)
            return [ocol(v.astype(np.int64), O.INT64) if cols[0] == O.INT64 else ocol(np.array([b"k%d" % x for x in v], dtype=object), O.STRING)]
        build, pr = keys(nb), keys(npr)
        if nb:
            build[0].valid[rng.random(nb) < 0.2] = False
        check_join(b2, build, pr, what=(cols, nb, npr))
        if nb:
            first = np.sort(np.unique(build[0].values, return_index=True)[1])
            check_join(b2, take(build, first), pr, what=(cols, nb, npr, "distinct"))


# ---- 4. inputs built against the table's own hash --------------------------------------------------------------------
def _collision_case(b2, build_a, probe_ab, filler, nb, what):
    """one key of each tag-sharing pair on the build side (plus filler up to nb rows), both keys probed"""
    build = build_a if filler is None else [O.OCol(_concat(a.values, f.values[: nb - len(a)]), np.ones(nb, bool), a.typ)
                                            for a, f in zip(build_a, filler)]
    want = join_maps_all(build, probe_ab, False)
    npairs = len(build_a[0])
    assert np.array_equal(want[SEMI][0][: npairs], np.arange(npairs)) and not np.isin(np.arange(npairs, 2 * npairs), want[SEMI][0]).any()
    check_join(b2, build, probe_ab, nulls_equal=(False,), what=what)


def _concat(a, b):
    if a.dtype == object or b.dtype == object:
        out = np.empty(len(a) + len(b), dtype=object)
        out[: len(a)], out[len(a):] = a, b
        return out
    return np.concatenate([a, b])


@pytest.mark.parametrize("nb", [0, BLOOM_ROWS], ids=["bloom_off", "bloom_on"])
def test_tag_collisions_packed(b2, nb):
    """distinct INT64 keys a, b with equal tags (so equal start slots): a on the build side, a and b probed.  b must match
    nothing, on the one-key probe (INNER), the single-pass probe (LEFT / FULL OUTER) and count + write (SEMI / ANTI)"""
    rng = np.random.default_rng(21)
    cand = np.unique(rng.integers(-2**63, 2**63 - 1, 1 << 20, dtype=np.int64))
    i, j = tag_collisions(hash_packed([(cand, O.INT64)]))
    assert len(i) >= 50
    a, b = cand[i], cand[j]
    rest = np.setdiff1d(cand, np.r_[a, b])
    filler = [ocol(rest, O.INT64)] if nb else None
    _collision_case(b2, [ocol(a, O.INT64)], [ocol(np.r_[a, b], O.INT64)], filler, nb, "packed")


def _random_strings(rng, n, length):
    raw = rng.integers(0, 256, (n, length), dtype=np.uint8)
    raw = np.unique(raw, axis=0)
    return raw, np.array([bytes(r) for r in raw], dtype=object)


@pytest.mark.parametrize("nb", [0, BLOOM_ROWS], ids=["bloom_off", "bloom_on"])
@pytest.mark.parametrize("shape", ["string8", "dec128_high_word", "i64_i32"])
def test_tag_collisions_generic(b2, shape, nb):
    """the same for the generic table: 8-byte STRING keys, DECIMAL128 keys that differ only in their high word (rows_equal
    must compare both words) and a two-column key"""
    rng = np.random.default_rng(22 + len(shape))
    m = 1 << 20
    if shape == "string8":
        raw, strs = _random_strings(rng, m, 8)
        tags = row_hash([("string", raw)])
        cols = lambda idx: [ocol(strs[idx], O.STRING)]                                                # noqa: E731
    elif shape == "dec128_high_word":
        hi = np.unique(rng.integers(-2**62, 2**62, m, dtype=np.int64)).view(np.uint64)
        w = np.stack([np.full(len(hi), 12345, np.uint64), hi], axis=1)
        tags = row_hash([("dec128", w)])
        cols = lambda idx: [ocol(w[idx], (O.DECIMAL128, 38, 0))]                                      # noqa: E731
    else:
        x = np.unique(rng.integers(-2**63, 2**63 - 1, m, dtype=np.int64))
        y = rng.integers(-2**31, 2**31, len(x)).astype(np.int32)
        tags = row_hash([("fixed", x, O.INT64), ("fixed", y, O.INT32)])
        cols = lambda idx: [ocol(x[idx], O.INT64), ocol(y[idx], O.INT32)]                             # noqa: E731
    i, j = tag_collisions(tags)
    assert len(i) >= 50
    rest = np.setdiff1d(np.arange(len(tags)), np.r_[i, j])
    _collision_case(b2, cols(i), cols(np.r_[i, j]), cols(rest) if nb else None, nb, shape)


def _keys_at_slots(layout, slots, mask, count, rng, exclude=()):
    """`count` keys (as id arrays for the layout's key columns) whose start slot is in `slots`"""
    found, seen = [], set(exclude)
    while sum(len(f) for f in found) < count:
        x = rng.integers(-2**63, 2**63 - 1, 1 << 21, dtype=np.int64)
        t = hash_packed([(x, O.INT64)]) if layout == "packed" else row_hash([("fixed", x, O.INT64), ("fixed", ~x, O.INT64)])
        x = x[np.isin(t & U64(mask), np.array(slots, dtype=np.uint64))]
        found.append(np.array([v for v in x.tolist() if v not in seen], dtype=np.int64))
        seen.update(found[-1].tolist())
    return np.concatenate(found)[:count]


def _layout_cols(layout, x):
    return [ocol(x, O.INT64)] if layout == "packed" else [ocol(x, O.INT64), ocol(~x, O.INT64)]


@pytest.mark.parametrize("nb", [500, BLOOM_ROWS], ids=["cap_1024", "cap_2^19_bloom"])
@pytest.mark.parametrize("layout", ["packed", "generic"])
def test_wrap_around_chains(b2, layout, nb):
    """keys whose start slot is one of the last three of the table, so their chains run past the end into slots 0, 1, ...
    which hold keys of their own; probed with every build key and with absent keys starting at the last slot"""
    rng = np.random.default_rng(31 + nb)
    cap = capacity(nb)
    mask = cap - 1
    tail = _keys_at_slots(layout, [cap - 3, cap - 2, cap - 1], mask, 12, rng)
    head = _keys_at_slots(layout, [0, 1, 2], mask, 6, rng, exclude=tail)
    absent = _keys_at_slots(layout, [cap - 1], mask, 8, rng, exclude=np.r_[tail, head])
    rest = np.setdiff1d(rng.integers(-2**63, 2**63 - 1, nb + 1000, dtype=np.int64), np.r_[tail, head, absent])[: nb - 18]
    bk = rng.permutation(np.r_[tail, head, rest])
    assert len(bk) == nb and capacity(len(bk)) == cap
    pk = np.r_[bk, absent, tail]
    check_join(b2, _layout_cols(layout, bk), _layout_cols(layout, pk), nulls_equal=(False,), what=(layout, nb))


@pytest.mark.parametrize("layout", ["packed", "generic"])
def test_long_chains(b2, layout):
    """300 distinct keys sharing one start slot (plus absent keys starting there), and one key on 5000 build rows"""
    rng = np.random.default_rng(41)
    same = _keys_at_slots(layout, [77], 1023, 400, rng)
    filler = np.setdiff1d(rng.integers(-2**63, 2**63 - 1, 300, dtype=np.int64), same)[:200]
    bk = rng.permutation(np.r_[same[:300], filler])
    assert capacity(len(bk)) == 1024
    pk = rng.permutation(np.r_[same, filler, same[:300]])
    check_join(b2, _layout_cols(layout, bk), _layout_cols(layout, pk), nulls_equal=(False,), what=(layout, "one slot"))
    hot = np.int64(-123456789)
    bk = rng.permutation(np.r_[np.full(5000, hot), filler])
    pk = rng.permutation(np.r_[np.full(40, hot), filler, same[:100]])
    check_join(b2, _layout_cols(layout, bk), _layout_cols(layout, pk), nulls_equal=(False,), what=(layout, "one key x 5000"))


# ---- 5. output past 2^31 - 1 rows -----------------------------------------------------------------------------------
def test_output_past_int32_rows_is_refused(b2):
    """64 keys with 1024 build rows and 32769 stream rows each: 2 147 549 184 pairs.  INNER raises B2_ERR_SIZE_OVERFLOW
    instead of returning a truncated map"""
    keys = key_of(np.arange(64))
    assert 64 * 1024 * 32769 > 2**31 - 1
    ht = b2.JoinHashTable(b2.Table.from_columns([b2.Column.from_numpy(np.repeat(keys, 1024))]))
    pt = b2.Table.from_columns([b2.Column.from_numpy(np.tile(keys, 32769))])
    with pytest.raises(b2.B2Error) as e:
        ht.probe(pt, INNER)
    assert e.value.code == ERR_SIZE_OVERFLOW


# ---- 6. the gather behind the join ------------------------------------------------------------------------------------
GATHER_TYPES = [O.BOOL8, O.INT8, O.INT16, O.INT32, O.INT64, (O.DECIMAL128, 30, 2), O.STRING]


def _payload(rng, typ, n, nullable):
    typ = typ if isinstance(typ, tuple) else (typ, 0, 0)
    dt = typ[0]
    if dt == O.STRING:
        v = np.array([b"s%d" % x * int(x % 4) for x in rng.integers(0, 1000, n)], dtype=object)
    elif dt == O.DECIMAL128:
        v = np.array([int(x) * 10**20 + int(y) for x, y in zip(rng.integers(-10**9, 10**9, n), rng.integers(0, 10**9, n))], dtype=object)
    elif dt == O.BOOL8:
        v = rng.integers(0, 2, n).astype(np.int8)
    else:
        v = rng.integers(-2**62, 2**62, n).astype(O._NP[dt])
    return O.OCol(v, (rng.random(n) > 0.2) if nullable else np.ones(n, bool), typ)


def test_gather_more_columns_than_one_launch(b2):
    """b2.gather of 70 fixed-width columns (two gather_fixed_kernel launches: at most 64 columns each) of every width plus
    STRING columns, nullable and not, by LEFT OUTER and FULL OUTER maps (out-of-bounds -> NULL) of 31, 32, 33 rows and in
    full"""
    from oracle import spark_relational as R
    from tests import datagen as G
    rng = np.random.default_rng(51)
    n = 300
    fixed_types = GATHER_TYPES[:-1]
    cols = [_payload(rng, fixed_types[k % len(fixed_types)], n, (k // len(fixed_types)) % 2 == 1) for k in range(70)]
    cols += [_payload(rng, O.STRING, n, k % 2 == 1) for k in range(4)]
    t = b2.Table.from_columns([G.to_b2_column(b2, c) for c in cols])
    bk = [ocol(rng.integers(0, 400, n).astype(np.int64), O.INT64)]
    pk = [ocol(rng.integers(0, 400, n).astype(np.int64), O.INT64)]
    ht = b2.JoinHashTable(to_table(b2, bk))
    b2.profile_enable(True)
    try:
        for kind in (LEFT_OUTER, FULL_OUTER):
            lm, rm = ht.probe(to_table(b2, pk), kind)
            for m in (lm, rm):
                full = m.to_numpy()[0]
                assert (full == INT32_MIN).any() or (kind == LEFT_OUTER and m is lm)
                for part in (full[:31], full[:32], full[:33], full[-31:], full[-32:], full[-33:], full):
                    out = b2.gather(t, b2.Column.from_numpy(part.astype(np.int32)), True)
                    want = R.gather(cols, part, True)
                    for c in range(len(cols)):
                        G.assert_col_equal(out.column(c), want[c])
        launches = {k["name"]: k["launches"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    assert launches.get("gather_fixed_kernel") == 2 * (2 * 2 * 7), launches       # two launches per gather


# ---- 7. the join exec -------------------------------------------------------------------------------------------------
def _exec_sides(rng):
    """stream: three batches (one empty) of [key INT64, f INT32, sid INT32, i16, i32 nullable, str nullable, dec128];
    build: two batches, the second with NULL keys and NULL payload, of [key INT64, bid INT32, i8, dec128, str]"""
    sizes = [(1 << 16) + 100, 0, 3000]
    ns = sum(sizes)
    nb1, nb2 = 3000, 2000
    ids = rng.permutation(4 * (nb1 + nb2))[: nb1 + nb2]
    bkey = key_of(ids)
    bvalid = np.r_[np.ones(nb1, bool), rng.random(nb2) > 0.2]
    build = [ocol(bkey, O.INT64, bvalid), ocol(np.arange(nb1 + nb2, dtype=np.int32), O.INT32),
             _payload(rng, O.INT8, nb1 + nb2, False), _payload(rng, (O.DECIMAL128, 30, 2), nb1 + nb2, False), _payload(rng, O.STRING, nb1 + nb2, False)]
    for c in build[2:]:
        c.valid[nb1:] = rng.random(nb2) > 0.3
    skey = key_of(np.where(rng.random(ns) < 0.5, rng.choice(ids, ns), 4 * (nb1 + nb2) + rng.integers(0, 1000, ns)))
    stream = [ocol(skey, O.INT64), ocol(rng.integers(0, 1000, ns).astype(np.int32), O.INT32), ocol(np.arange(ns, dtype=np.int32), O.INT32),
              _payload(rng, O.INT16, ns, False), _payload(rng, O.INT32, ns, True), _payload(rng, O.STRING, ns, True),
              _payload(rng, (O.DECIMAL128, 30, 2), ns, False)]
    bounds = np.cumsum([0] + sizes)
    stream[1].values[bounds[2]:] = rng.integers(0, 500, sizes[2])       # the filter passes no row of the last batch
    sbatches = [take(stream, np.arange(bounds[i], bounds[i + 1])) for i in range(3)]
    bbatches = [take(build, np.arange(0, nb1)), take(build, np.arange(nb1, nb1 + nb2))]
    return stream, build, sbatches, bbatches


def _column_arrays(col):
    v, ok = col.to_numpy()
    return list(v), ok


@pytest.mark.parametrize("prune", [False, True], ids=["all_columns", "pruned"])
@pytest.mark.parametrize("filtered", [False, True], ids=["no_filter", "filter_below"])
@pytest.mark.parametrize("kind", KINDS)
def test_join_exec(b2, kind, filtered, prune):
    """GpuShuffledHashJoinExec over batches against the reference maps gathered in numpy; with a GpuFilterExec below the
    stream (fused through a selection vector, or for INNER into the probe itself; it passes no row of the last batch, an
    empty selection vector) and with column pruning"""
    from oracle import spark_relational as R
    from spark_rapids_b200 import execs as E
    rng = np.random.default_rng(61)
    stream, build, sbatches, bbatches = _exec_sides(rng)
    src = E.GpuBatchSource([to_table(b2, s) for s in sbatches])
    keep = np.ones(len(stream[0]), bool)
    if filtered:
        keep = stream[1].values >= 500
        src = E.GpuFilterExec(b2.col(1, b2.INT32, nullable=False) >= b2.lit(500, b2.INT32), src)
    so, bo = ([2, 0, 5, 6, 3], [1, 3, 4, 2]) if prune else (list(range(len(stream))), list(range(len(build))))
    kw = dict(stream_out=so, build_out=bo) if prune else {}
    j = E.GpuShuffledHashJoinExec([0], [0], kind, src, E.GpuBatchSource([to_table(b2, b) for b in bbatches]), **kw)
    b2.profile_enable(True)
    try:
        out = j.collect()
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    if kind == INNER and filtered:
        assert "join_filter_probe_kernel" in names, names
    rows = np.flatnonzero(keep)
    lm, rm = join_maps(build[:1], take(stream[:1], rows), kind)
    lm = np.where(lm >= 0, rows[np.maximum(lm, 0)], INT32_MIN)
    want = R.gather([stream[c] for c in so], lm, True)
    if kind not in (SEMI, ANTI):
        want += R.gather([build[c] for c in bo], rm, True)
    got = [out.column(c) for c in range(out.num_columns)]
    assert len(got) == len(want) and out.num_rows == len(lm)
    sid_at, bid_at = so.index(2), len(so) + bo.index(1)                     # the row-id columns order both sides
    def order(vals, valid):
        s = np.where(valid[sid_at], np.asarray(vals[sid_at], np.int64), -1)
        if kind in (SEMI, ANTI):
            return np.argsort(s, kind="stable")
        return np.lexsort((np.where(valid[bid_at], np.asarray(vals[bid_at], np.int64), -1), s))
    gv = [_column_arrays(c) for c in got]
    og = order([v for v, _ in gv], [ok for _, ok in gv])
    ow = order([c.values for c in want], [c.valid for c in want])
    for (v, ok), w in zip(gv, want):
        assert np.array_equal(ok[og], w.valid[ow])
        gvals = [x for x, k in zip(np.asarray(v, dtype=object)[og], ok[og]) if k]
        wvals = [x for x, k in zip(np.asarray(w.values, dtype=object)[ow], w.valid[ow]) if k]
        assert [int(x) if not isinstance(x, bytes) else x for x in gvals] == [int(x) if not isinstance(x, bytes) else x for x in wvals]
