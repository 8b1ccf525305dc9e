"""The shuffle's data paths against exact references: the B2T1 wire format (csrc/serialize.cu) written at every validity bit
offset and read back from mixed writers, malformed descriptors rejected, the JCUDF row conversion (csrc/rows.cu) in each
direction at every tile size it picks, and the fused hash exchange (csrc/exchange.cu) in a world of one, where the scatter
kernel stores into the rank's own arena: key modes, selection vectors, column pruning, validity bytes and the grow-and-retry
loop of an overflowing region."""
import numpy as np
import pytest

from oracle import shuffle_format as F
from oracle import spark_cpu as O
from tests import movement_reference as M

pytestmark = pytest.mark.gpu
TYPES = M.FIXED_TYPES + [O.STRING]


def _cols(rng, n, null_frac=0.3):
    return [M.rand_col(rng, dt, n, null_frac=null_frac if k % 2 else 0.0) for k, dt in enumerate(TYPES)]


def _check(got_cols, exp_cols, what, payload="valid", nullability=True):
    assert len(got_cols) == len(exp_cols), what
    for i, (g, e) in enumerate(zip(got_cols, exp_cols)):
        M.assert_same(g, e, "%s col %d" % (what, i), payload=payload, nullability=nullability)


# ---- serialise --------------------------------------------------------------------------------------------------------------
def test_serialize_every_bit_offset(b2):
    rng = np.random.default_rng(1)
    n = 90
    cols = _cols(rng, n, null_frac=0.4)
    t = M.to_table(b2, cols)
    for start in range(9):
        for end in (start, start + 1, start + 9, start + 33, n):
            raw = b2.serialize_table(t, start, end)
            assert len(raw) % 64 == 0 and M.header(raw) == (len(cols), end - start, len(raw))
            exp = [M.slice_col(c, start, end) for c in cols]
            _check([M.raw_of_ocol(p) for p in F.parse(raw)], exp, "slice [%d, %d)" % (start, end), nullability=False)
            for i, e in enumerate(exp):
                d = M.desc(raw, i)
                nulls = int((~e.valid_or_ones()).sum())
                assert d["null_count"] == nulls and d["validity_bytes"] == ((end - start + 7) // 8 if nulls else 0), (start, end, i, d)


def test_serialize_edge_columns(b2):
    """an all-NULL column, a nullable column whose slice holds no NULL (validity omitted), all-empty strings (no data
    bytes) and a zero-row slice"""
    rng = np.random.default_rng(2)
    n = 50
    all_null = M.rand_fixed(rng, O.INT64, n, null_frac=0.5)
    all_null.valid[:] = False
    holes = M.rand_fixed(rng, O.DECIMAL128, n, null_frac=0.5)
    holes.valid[:] = True
    holes.valid[[0, 49]] = False
    empty = M.rand_strings(rng, n, null_frac=0.3, empty_frac=1.0)
    cols = [all_null, holes, empty]
    t = M.to_table(b2, cols)
    for a, b in [(0, n), (1, 49), (3, 3), (n, n)]:
        raw = b2.serialize_table(t, a, b)
        d = [M.desc(raw, i) for i in range(3)]
        assert d[0]["null_count"] == b - a and d[0]["validity_bytes"] == ((b - a + 7) // 8 if b > a else 0)
        assert d[1]["null_count"] == (b - a) - int(holes.valid[a:b].sum()) and (d[1]["validity_bytes"] == 0) == (d[1]["null_count"] == 0)
        assert d[2]["data_bytes"] == 0 and d[2]["offsets_bytes"] == 4 * (b - a + 1)
        _check([M.raw_of_ocol(p) for p in F.parse(raw)], [M.slice_col(c, a, b) for c in cols], "[%d, %d)" % (a, b), nullability=False)
        back = M.from_table(b2, b2.deserialize_concat([raw]))
        _check(back, [M.slice_col(c, a, b) for c in cols], "round trip [%d, %d)" % (a, b), nullability=False)


# ---- coalesce on read -------------------------------------------------------------------------------------------------------
def _mixed_inputs(b2, rng, sizes, nullable):
    """per input: its columns, and its buffer from the GPU writer or the oracle writer (alternately).  The GPU writer
    serialises rows [2, 2 + n) of a table with more rows on either side, so its slice starts at bit 2."""
    parts, bufs = [], []
    for k, (sz, nl) in enumerate(zip(sizes, nullable)):
        cols = _cols(rng, sz, null_frac=0.4 if nl else 0.0)
        if k % 2 == 0:
            padded = [M.concat([M.rand_col(rng, c.dtype, 2, null_frac=0.5 if nl else 0.0), c,
                                M.rand_col(rng, c.dtype, 3, null_frac=0.5 if nl else 0.0)]) for c in cols]
            bufs.append(b2.serialize_table(M.to_table(b2, padded), 2, 2 + sz))
        else:
            bufs.append(np.frombuffer(F.build([M.ocol_of_raw(c) for c in cols]), np.uint8).copy())
        parts.append(cols)
    return parts, bufs


def test_coalesce_mixed_validity_and_writers(b2):
    """12 inputs: byte-aligned starts (whole validity bytes copied), unaligned starts (bit by bit), inputs without
    validity, zero-row inputs; buffers from the GPU writer and the oracle writer alternately"""
    rng = np.random.default_rng(3)
    sizes = [8, 5, 16, 3, 0, 7, 24, 1, 9, 2, 40, 13]
    nullable = [1, 1, 0, 1, 1, 1, 0, 1, 1, 0, 1, 1]
    parts, bufs = _mixed_inputs(b2, rng, sizes, nullable)
    got = M.from_table(b2, b2.deserialize_concat(bufs))
    exp = [M.concat([p[i] for p in parts]) for i in range(len(TYPES))]
    _check(got, exp, "coalesce", nullability=False)
    for g, e in zip(got, exp):   # validity is carried iff some row is NULL
        assert (g.valid is not None) == bool((~e.valid_or_ones()).any())


def _set_validity_padding(buf, col):
    """set every bit past the last row in the validity bytes of column `col` (a writer is not obliged to clear them)"""
    _, rows, _ = M.header(buf)
    d, off = M.desc(buf, col), M.buffer_offsets(buf)[col]["validity"]
    assert d["validity_bytes"] and rows & 7
    buf[off + d["validity_bytes"] - 1] |= (0xff << (rows & 7)) & 0xff


def test_coalesce_ignores_validity_padding_bits(b2):
    """inputs whose validity padding bits are set, each followed by an input whose first rows are NULL: the padding must
    not make those rows valid, whether the padded input was copied as whole bytes (it starts on a byte boundary) or bit by
    bit"""
    rng = np.random.default_rng(4)
    for sizes in ([13, 6, 11], [3, 13, 6, 11], [8, 13, 6, 11], [5, 3, 8, 2]):
        parts, bufs = [], []
        for k, sz in enumerate(sizes):
            cols = [M.rand_col(rng, dt, sz, null_frac=0.3) for dt in TYPES]
            for c in cols:
                c.valid[:1 if k == 0 else 2] = False
            cols = [M.take(c, np.arange(sz)) for c in cols]   # a NULL string holds no chars
            buf = np.frombuffer(F.build([M.ocol_of_raw(c) for c in cols]), np.uint8).copy()
            if sz & 7:
                for i in range(len(cols)):
                    _set_validity_padding(buf, i)
            parts.append(cols)
            bufs.append(buf)
        got = M.from_table(b2, b2.deserialize_concat(bufs))
        exp = [M.concat([p[i] for p in parts]) for i in range(len(TYPES))]
        _check(got, exp, "padding bits, input sizes %s" % sizes)


def _bad_buffer_cases(good):
    """(name, mutate(buf)) for every descriptor inconsistency; good = INT64 nullable, STRING nullable, INT32, DECIMAL128"""
    _, n, _ = M.header(good)
    offs = M.buffer_offsets(good)
    d = [M.desc(good, i) for i in range(4)]
    so = offs[1]["offsets"]

    def setd(col, field, value):
        return lambda b: M.set_desc(b, col, field, value)

    def set_off(i, v):
        def f(b):
            b[so + 4 * i:so + 4 * i + 4] = np.frombuffer(np.int32(v).tobytes(), np.uint8)
        return f

    str_offs = np.frombuffer(good, np.int32, n + 1, so)
    k = int(np.flatnonzero(np.diff(str_offs) > 0)[3]) + 1   # an interior offset with a longer string before it
    return [
        ("validity_bytes 0 with NULLs", setd(0, "validity_bytes", 0)),
        ("validity_bytes short", setd(0, "validity_bytes", d[0]["validity_bytes"] - 1)),
        ("validity_bytes long", setd(0, "validity_bytes", d[0]["validity_bytes"] + 64)),
        ("validity_bytes on a column without NULLs", setd(2, "validity_bytes", (n + 7) // 8)),
        ("validity_bytes negative", setd(0, "validity_bytes", -64)),
        ("null_count negative", setd(0, "null_count", -1)),
        ("null_count above rows", setd(0, "null_count", n + 1)),
        ("null_count disagrees with the bits", setd(0, "null_count", d[0]["null_count"] + 1)),
        ("offsets_bytes short", setd(1, "offsets_bytes", 4 * n)),
        ("offsets_bytes long", setd(1, "offsets_bytes", 4 * (n + 1) + 64)),
        ("offsets_bytes negative", setd(1, "offsets_bytes", -4)),
        ("offsets_bytes on a fixed-width column", setd(2, "offsets_bytes", 4 * (n + 1))),
        ("data_bytes 0 for INT64 rows", setd(0, "data_bytes", 0)),
        ("data_bytes short", setd(3, "data_bytes", 16 * n - 16)),
        ("data_bytes long", setd(2, "data_bytes", 4 * n + 64)),
        ("data_bytes negative (fixed)", setd(2, "data_bytes", -4)),
        ("data_bytes negative (string)", setd(1, "data_bytes", -8)),
        ("data_bytes past the buffer (string)", setd(1, "data_bytes", 1 << 40)),
        ("string offsets do not start at 0", set_off(0, 1)),
        ("string offsets decrease", set_off(k, int(str_offs[k - 1]) - 1)),
        ("string offsets end before data_bytes", set_off(n, d[1]["data_bytes"] - 1)),
        ("string offsets end after data_bytes", set_off(n, d[1]["data_bytes"] + 1)),
        ("unknown dtype", setd(2, "dtype", 13)),
        ("rows disagree with every descriptor", lambda b: M.set_header(b, "rows", n + 8)),
        ("header claims more columns than the buffer holds", lambda b: M.set_header(b, "ncols", 1000)),
        ("total_bytes inside the descriptors", lambda b: M.set_header(b, "total_bytes", 64)),
    ]


def test_malformed_descriptors_are_rejected(b2):
    """each buffer is a view of a larger array, so even a reader that trusts the descriptor only reads memory that exists"""
    rng = np.random.default_rng(5)
    n = 100
    cols = [M.rand_fixed(rng, O.INT64, n, null_frac=0.3), M.rand_strings(rng, n, null_frac=0.2, empty_frac=0.1),
            M.rand_fixed(rng, O.INT32, n), M.rand_fixed(rng, O.DECIMAL128, n)]
    good = np.frombuffer(F.build([M.ocol_of_raw(c) for c in cols]), np.uint8).copy()
    spare = 1 << 17
    ok = M.from_table(b2, b2.deserialize_concat([good]))
    _check(ok, cols, "the untouched buffer", nullability=False)
    small = [M.rand_fixed(rng, O.INT64, 7, 0.5), M.rand_strings(rng, 7), M.rand_fixed(rng, O.INT32, 7), M.rand_fixed(rng, O.DECIMAL128, 7)]
    other = np.frombuffer(F.build([M.ocol_of_raw(c) for c in small]), np.uint8).copy()
    for name, mutate in _bad_buffer_cases(good):
        big = np.zeros(len(good) + spare, np.uint8)
        big[:len(good)] = good
        view = big[:len(good)]
        mutate(view)
        for inputs in ([view], [other, view], [view, other]):
            with pytest.raises(b2.B2Error):
                b2.deserialize_concat(inputs)
                pytest.fail("accepted: %s" % name)


def test_mismatched_inputs_are_rejected(b2):
    rng = np.random.default_rng(6)

    def buf(cols):
        return np.frombuffer(F.build([M.ocol_of_raw(c) for c in cols]), np.uint8).copy()

    a = buf([M.rand_fixed(rng, O.INT64, 9), M.rand_fixed(rng, O.DECIMAL64, 9)])
    fewer = buf([M.rand_fixed(rng, O.INT64, 9)])
    other_type = buf([M.rand_fixed(rng, O.INT64, 9), M.rand_fixed(rng, O.FLOAT64, 9)])
    other_scale = buf([M.rand_fixed(rng, O.INT64, 9), M.Raw(O.DECIMAL64, M.rand_fixed(rng, O.DECIMAL64, 9).data, scale=3)])
    assert M.from_table(b2, b2.deserialize_concat([a, a]))[0].data.shape == (18, 8)
    for bad in ([a, fewer], [fewer, a], [a, other_type], [a, other_scale]):
        with pytest.raises(b2.B2Error):
            b2.deserialize_concat(bad)


# ---- JCUDF rows -------------------------------------------------------------------------------------------------------------
def _layout(ncols, kind):
    if kind == "narrow":
        return [[O.INT8, O.BOOL8, O.INT16, O.INT32, O.FLOAT32][k % 5] for k in range(ncols)]
    if kind == "wide":
        return [O.DECIMAL128] * ncols
    return [M.FIXED_TYPES[(3 * k) % len(M.FIXED_TYPES)] for k in range(ncols)]


_LAYOUTS = [(1, "narrow"), (8, "narrow"), (9, "mixed"), (16, "narrow"), (17, "mixed"), (64, "narrow"), (40, "mixed"), (64, "wide"),
            (1, "wide"), (9, "wide")]


def _row_sizes(dtypes):
    rb = M.row_layout(dtypes)[2]
    rpt = M.rows_per_tile(rb)
    # the grid holds up to 2 CTAs per SM (264 on an H100): enough tiles that every CTA loops, within ~64 MB of rows
    big = min(600 * rpt, (64 << 20) // rb)
    return rb, rpt, [rpt - 1, rpt, rpt + 1, big]


def test_row_layouts_cover_every_tile_size():
    tiles = sorted({M.rows_per_tile(M.row_layout(_layout(nc, kind))[2]) for nc, kind in _LAYOUTS})
    assert tiles[0] == 64 and tiles[-1] == 1024 and len(tiles) >= 4, tiles


@pytest.mark.parametrize("ncols,kind", _LAYOUTS)
def test_to_rows(b2, ncols, kind):
    """validity bytes and valid payloads exact; alignment gaps, unused validity bits and the tail zero"""
    dtypes = _layout(ncols, kind)
    rb, rpt, sizes = _row_sizes(dtypes)
    rng = np.random.default_rng(ncols * 3 + len(kind))
    for n in sizes:
        cols = [M.rand_fixed(rng, dt, n, null_frac=0.3 if k % 3 != 1 else 0.0) for k, dt in enumerate(dtypes)]
        got = b2.table_to_rows(M.to_table(b2, cols))
        assert got.shape == (n, rb), (got.shape, n, rb)
        exp, defined = M.to_rows(cols), M.defined_bytes(cols)
        bad = np.flatnonzero((got != exp) & defined)
        assert not len(bad), "n=%d rpt=%d: %d bytes differ, first at row %d byte %d" % (n, rpt, len(bad), bad[0] // rb, bad[0] % rb)


@pytest.mark.parametrize("ncols,kind", _LAYOUTS)
def test_from_rows(b2, ncols, kind):
    """rows of random bytes: NULL fields, gaps, unused validity bits and the tail hold garbage the reader must ignore"""
    dtypes = _layout(ncols, kind)
    rb, rpt, sizes = _row_sizes(dtypes)
    rng = np.random.default_rng(ncols * 5 + len(kind))
    for n in sizes:
        rows = rng.integers(0, 256, (n, rb), dtype=np.uint8)
        got = M.from_table(b2, b2.table_from_rows(rows, dtypes))
        _check(got, M.from_rows(rows, dtypes), "n=%d rpt=%d" % (n, rpt))


def test_rows_round_trip(b2):
    rng = np.random.default_rng(7)
    dtypes = _layout(17, "mixed")
    cols = [M.rand_fixed(rng, dt, 5000, null_frac=0.2) for dt in dtypes]
    back = M.from_table(b2, b2.table_from_rows(b2.table_to_rows(M.to_table(b2, cols)), dtypes, [0] * 17))
    _check(back, cols, "round trip")


def test_rows_reject_unsupported_tables(b2):
    rng = np.random.default_rng(8)
    wide = M.to_table(b2, [M.rand_fixed(rng, O.INT8, 4) for _ in range(65)])
    with pytest.raises(b2.B2Error):
        b2.table_to_rows(wide)
    with pytest.raises(b2.B2Error):
        b2.table_to_rows(M.to_table(b2, [M.rand_fixed(rng, O.INT32, 4), M.rand_strings(rng, 4)]))
    with pytest.raises(b2.B2Error):
        b2.table_from_rows(np.zeros((4, 72), np.uint8), [O.INT8] * 65)
    with pytest.raises(b2.B2Error):
        b2.table_from_rows(np.zeros((4, 16), np.uint8), [O.INT32, O.STRING])


# ---- fused exchange, world of one -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def comm(b2):
    c = b2.Comm(b2.Comm.unique_id(), 0, 1)
    assert c.fused_ready()
    yield c
    c.close()


def _exchange(b2, comm, cols, keys, sel=None, out_cols=None):
    """send `cols` plus a row-id column (always travelling, last) -> (received Raw columns, ids); checks the rows exactly"""
    n = len(cols[0])
    ids = M.Raw(O.INT32, data=np.arange(n, dtype=np.int32).view(np.uint8).reshape(n, 4))
    full = cols + [ids]
    travel = list(range(len(cols))) if out_cols is None else list(out_cols)
    t = M.to_table(b2, full)
    sel_col = None if sel is None else b2.Column.from_numpy(np.asarray(sel, np.int32))
    out, anyd = comm.exchange_hash_sel(t, keys, sel_col, travel + [len(cols)])
    assert anyd and out is not None
    got = M.from_table(b2, out)
    picked = np.arange(n) if sel is None else np.asarray(sel, np.int64)
    rid = got[-1].data.view(np.int32).reshape(-1).astype(np.int64)
    # a world of one receives every selected row once, in an order the exchange does not promise
    assert np.array_equal(np.sort(rid), np.sort(picked)), "rows lost or duplicated"
    exp = [M.take(full[c], rid) for c in travel]
    _check(got[:-1], exp, "exchange keys=%s" % (keys,))
    return got


@pytest.mark.parametrize("key_type", [O.INT64, O.TIMESTAMP_US, O.DECIMAL64, O.INT32, O.DATE32])
def test_exchange_integer_key_modes(b2, comm, key_type):
    """one non-null 8-byte key (the 64-bit key mode) or 4-byte key (the 32-bit key mode)"""
    rng = np.random.default_rng(key_type)
    n = 9000
    cols = [M.rand_fixed(rng, key_type, n)] + _cols(rng, n)[:-1]
    _exchange(b2, comm, cols, [0])


def test_exchange_generic_key_mode(b2, comm):
    """the generic key mode: a nullable key, two keys, a STRING key that does not travel, no keys (SinglePartition)"""
    rng = np.random.default_rng(9)
    n = 5000
    cols = [M.rand_fixed(rng, O.INT64, n, null_frac=0.3), M.rand_strings(rng, n, null_frac=0.2), M.rand_fixed(rng, O.INT32, n),
            M.rand_fixed(rng, O.DECIMAL128, n, null_frac=0.1), M.rand_fixed(rng, O.FLOAT32, n)]
    fixed = [0, 2, 3, 4]
    for keys in ([0], [2, 3], [1], [1, 0], []):
        _exchange(b2, comm, cols, keys, out_cols=fixed)


@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, 3 * 4096 + 5])
def test_exchange_tile_edges_every_width(b2, comm, n):
    rng = np.random.default_rng(n)
    cols = _cols(rng, n)[:-1]
    _exchange(b2, comm, cols, [4])


def test_exchange_selection_and_pruning(b2, comm):
    rng = np.random.default_rng(10)
    n = 11000
    cols = _cols(rng, n)[:-1] + [M.rand_strings(rng, n)]
    string_col = len(cols) - 1
    for frac in (0.0, 0.001, 0.5, 1.0):
        sel = np.flatnonzero(rng.random(n) < frac)
        for out_cols in ([9, 0, 5, 2], [3], list(range(string_col))[::-1]):
            _exchange(b2, comm, cols, [string_col, 6], sel=sel, out_cols=out_cols)


def test_exchange_column_limits(b2, comm):
    rng = np.random.default_rng(11)
    n = 300
    cols = [M.rand_fixed(rng, M.FIXED_TYPES[k % len(M.FIXED_TYPES)], n, null_frac=0.2 if k % 2 else 0.0) for k in range(31)]
    _exchange(b2, comm, cols, [0, 7])   # 31 + the id column: the 32-column limit
    ids = M.Raw(O.INT32, data=np.arange(n, dtype=np.int32).view(np.uint8).reshape(n, 4))
    too_many = M.to_table(b2, cols + [ids, ids])
    with pytest.raises(b2.B2Error):
        comm.exchange_hash_sel(too_many, [0])
    with pytest.raises(b2.B2Error):
        comm.exchange_hash_sel(M.to_table(b2, [cols[0], M.rand_strings(rng, n)]), [0])
    with pytest.raises(b2.B2Error):
        comm.exchange_hash_sel(M.to_table(b2, cols[:3]), [0], out_cols=[0, 3])


def test_exchange_without_a_batch(b2, comm):
    out, anyd = comm.exchange_hash_sel(None, [0])
    assert out is None and not anyd


def test_exchange_grows_an_overflowing_arena(b2, monkeypatch):
    """a 1 MB arena: the first store overflows its region, the arenas grow and the call is retried; a second call on the
    grown arenas (the other parity) is exact too"""
    monkeypatch.setenv("B2_EXCHANGE_ARENA_MB", "1")
    c = b2.Comm(b2.Comm.unique_id(), 0, 1)
    try:
        assert c.fused_ready() and c.stats()["arena_bytes"] == 1 << 20
        rng = np.random.default_rng(12)
        for n in (200_000, 70_000):
            cols = [M.rand_fixed(rng, O.INT64, n, null_frac=0.3), M.rand_fixed(rng, O.DECIMAL128, n), M.rand_fixed(rng, O.INT8, n, 0.5)]
            _exchange(b2, c, cols, [0])
        assert c.stats()["arena_bytes"] > 1 << 20
    finally:
        c.close()
