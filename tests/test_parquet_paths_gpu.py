"""Every decode path of csrc/parquet.cu against pyarrow (oracle.spark_parquet), exactly: dtype, scale, validity and
values, floats bit for bit (NaN payloads, -0.0, +-inf).

 A. pyarrow-written files: every supported physical / logical type (unsigned ints as the signed view of their width,
    TIMESTAMP millis and micros, decimals as INT32 / INT64 / FIXED_LEN_BYTE_ARRAY at precisions 1 to 38), dictionary
    on / off / falling back to PLAIN part way through a chunk, V1 / V2 pages, none / snappy, 1 KiB pages up to pages
    above the 192 KiB threshold of snappy_big_kernel, several row groups, REQUIRED and OPTIONAL fields, and NULL
    patterns (none, 15 %, 99 %, all, 2000-row NULL runs); dictionaries of 1 to 2^18 + 1 entries.
 B. hand-built pages (tests/parquet_pages.py): the shapes pyarrow never writes.
 C. malformed input: truncated level / index streams, over-claiming runs, bad level lengths, short pages -> B2_ERR_INVALID
    and no device bytes left in use; encodings, codecs and types outside the decoder -> B2_ERR_UNSUPPORTED.
Which kernels ran is read from the kernel timings; `parquet_last_stats()` shows pages read in place."""
import decimal
import io
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle import spark_cpu as O
from oracle import spark_parquet as P
from tests import parquet_pages as W

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = 1, 5
SHAPES = W.all_shapes()


def _decode(b2, raw, cols):
    """-> (table, names of the kernels the decode launched)"""
    b2.profile_enable(True)
    try:
        t = b2.parquet_decode(raw, cols)
        names = {k["name"] for k in b2.profile_report()}
    finally:
        b2.profile_enable(False)
    return t, names


def _assert_exact(got, oc, what):
    dt, _, scale = oc.typ
    assert (got.dtype, len(got)) == (dt, len(oc)), (what, got.dtype, dt, len(got), len(oc))
    if O.is_decimal(dt):
        assert got.scale == scale, (what, got.scale, scale)
    vals, valid = got.to_numpy()
    assert np.array_equal(valid, oc.valid), (what, "validity", np.flatnonzero(valid != oc.valid)[:5])
    v = oc.valid
    if dt in (O.FLOAT32, O.FLOAT64):
        ut = np.uint32 if dt == O.FLOAT32 else np.uint64
        exp = np.asarray(oc.values, dtype=O._NP[dt]).view(ut)
        bad = np.flatnonzero(v & (vals.view(ut) != exp))
    elif dt == O.STRING or dt == O.DECIMAL128:
        bad = [i for i in np.flatnonzero(v) if vals[i] != oc.values[i]]
    else:
        bad = np.flatnonzero(v & (vals.astype(np.int64) != np.asarray(oc.values).astype(np.int64)))
    assert len(bad) == 0, (what, [(int(i), vals[i], oc.values[i]) for i in bad[:5]])


def _check(b2, raw, cols, float_bits=None):
    t, names = _decode(b2, raw, cols)
    exp = P.read_parquet(raw, cols)
    for i, c in enumerate(cols):
        _assert_exact(t.column(i), exp[i], c)
    if float_bits:   # the oracle goes through Python floats: pin the payloads against the written bits as well
        for c, bits in float_bits.items():
            vals, valid = t.column(cols.index(c)).to_numpy()
            assert np.array_equal(vals.view(bits.dtype)[valid], bits[valid]), c
    return t, names


# ---- A. pyarrow-written files ---------------------------------------------------------------------------------------
F32_SPECIAL = np.array([0x7FC00000, 0x7FC12345, 0xFFC00001, 0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x00000001], np.uint32)
F64_SPECIAL = np.array([0x7FF8000000000000, 0x7FF8DEADBEEF0001, 0xFFF8000000000007, 1 << 63, 0, 0x7FF0000000000000,
                        0xFFF0000000000000, 1], np.uint64)
DEC_PRECISIONS = (1, 2, 3, 9, 10, 18, 19, 28, 38)


def _decimals(p, n, rng):
    """±(10^p − 1), 0, ±1, the values where the two's-complement byte length changes, then random digits"""
    lim = 10 ** p - 1
    edges = [lim, -lim, 0, 1, -1]
    for b in range(1, 17):
        for v in (2 ** (8 * b - 1) - 1, 2 ** (8 * b - 1), -(2 ** (8 * b - 1)), -(2 ** (8 * b - 1)) - 1):
            if abs(v) <= lim:
                edges.append(v)
    vals = [int(x) % (2 * lim + 1) - lim for x in rng.integers(0, 2**62, n)]
    vals[:len(edges)] = edges[:n]
    return vals


def _mask(n, rng, nulls):
    if nulls == "none":
        return None
    if nulls == "all":
        return np.ones(n, bool)
    if nulls == "runs":   # 2000-row NULL runs: whole NULL pages between full ones under the 1 KiB writers, one run inside a page otherwise
        return ((np.arange(n) // 2000) % 3) == 1
    return rng.random(n) < {"15": 0.15, "99": 0.99}[nulls]


def matrix_table(n, rng, nulls, required=False):
    """one column of every type the decoder supports; -> (table, {float column: written bits})"""
    cols, bits, fields = {}, {}, []

    def add(name, values, typ, cast=None):
        m = None if required else _mask(n, rng, nulls)
        a = pa.array(values, typ, mask=m)
        cols[name] = a.cast(cast) if cast is not None else a
        fields.append(pa.field(name, cols[name].type, nullable=not required))

    ints = {"i8": (pa.int8(), np.int8), "i16": (pa.int16(), np.int16), "i32": (pa.int32(), np.int32), "i64": (pa.int64(), np.int64),
            "u8": (pa.uint8(), np.uint8), "u16": (pa.uint16(), np.uint16), "u32": (pa.uint32(), np.uint32), "u64": (pa.uint64(), np.uint64)}
    for name, (typ, npt) in ints.items():
        info = np.iinfo(npt)
        v = rng.integers(info.min, info.max, n, endpoint=True, dtype=npt)
        v[:4] = [info.min, info.max, 0, 1 if info.min == 0 else -1]
        add(name, v, typ)
    add("b", rng.integers(0, 2, n).astype(bool), pa.bool_())
    f32 = rng.standard_normal(n).astype(np.float32).view(np.uint32)
    f32[:len(F32_SPECIAL)] = F32_SPECIAL
    f64 = (rng.standard_normal(n) * 1e300).view(np.uint64)
    f64[:len(F64_SPECIAL)] = F64_SPECIAL
    add("f32", f32.view(np.float32), pa.float32())
    add("f64", f64.view(np.float64), pa.float64())
    bits["f32"], bits["f64"] = f32, f64
    add("date", rng.integers(-100000, 100000, n).astype(np.int32), pa.int32(), pa.date32())
    add("ts_us", rng.integers(-2**55, 2**57, n), pa.int64(), pa.timestamp("us"))     # years 829 to 6536: Python datetimes
    add("ts_ms", rng.integers(-2**45, 2**47, n), pa.int64(), pa.timestamp("ms"))
    for p in DEC_PRECISIONS:
        s = min(p, 2)
        exact = decimal.Context(prec=80)
        add("dec%d" % p, [decimal.Decimal(v).scaleb(-s, exact) for v in _decimals(p, n, rng)], pa.decimal128(p, s))
    words = ["", "a", "é", "日本語", "x" * 100, "ÿĀ", "long " * 300]
    add("s", [words[i % len(words)] + ("%d" % i if i % 5 else "") for i in rng.integers(0, 10**6, n)], pa.string())
    return pa.table(cols, schema=pa.schema(fields)), bits


def _write(tbl, **kw):
    sink = io.BytesIO()
    pq.write_table(tbl, sink, **kw)
    return sink.getvalue()


WRITERS = {
    "plain_none_v1": dict(compression="none", use_dictionary=False),
    "dict_snappy_v1": dict(compression="snappy", use_dictionary=True),
    "dict_snappy_v2_1k": dict(compression="snappy", use_dictionary=True, data_page_version="2.0", data_page_size=1024, write_batch_size=64),
    "plain_snappy_v2": dict(compression="snappy", use_dictionary=False, data_page_version="2.0"),
    "fallback_snappy_1k": dict(compression="snappy", use_dictionary=True, dictionary_pagesize_limit=2048, data_page_size=1024,
                               write_batch_size=64),
    "fallback_none_v2": dict(compression="none", use_dictionary=True, dictionary_pagesize_limit=4096, data_page_version="2.0"),
    "int_decimals_rg": dict(compression="snappy", store_decimal_as_integer=True, row_group_size=2500, data_page_size=4096),
    "big_pages": dict(compression="snappy", use_dictionary=False, data_page_size=400 << 10, max_rows_per_page=1 << 20),
}
NULLS = ["none", "15", "99", "all", "runs"]


@pytest.mark.parametrize("nulls", NULLS)
@pytest.mark.parametrize("writer", sorted(WRITERS))
def test_matrix_vs_pyarrow(b2, writer, nulls):
    n = 6000
    tbl, bits = matrix_table(n, np.random.default_rng(len(writer) * 7 + len(nulls)), nulls)
    raw = _write(tbl, **WRITERS[writer])
    t, names = _check(b2, raw, tbl.column_names, bits if nulls == "none" else None)
    assert t.num_rows == n and {"values_kernel", "levels_kernel"} <= names, names
    if nulls in ("15", "99", "runs"):
        assert {"expand_nulls_kernel", "expand_null_lengths_kernel", "string_chars_kernel"} <= names, names
    if writer == "big_pages" and nulls in ("none", "15", "runs"):   # the string column's pages are above 192 KiB
        assert "snappy_big_kernel" in names, names


@pytest.mark.parametrize("writer", ["plain_none_v1", "dict_snappy_v2_1k", "fallback_snappy_1k", "int_decimals_rg"])
def test_required_fields(b2, writer):
    """REQUIRED columns: no definition levels, no levels kernel, values straight from the page start"""
    tbl, bits = matrix_table(5000, np.random.default_rng(3), "none", required=True)
    raw = _write(tbl, **WRITERS[writer])
    assert pq.ParquetFile(io.BytesIO(raw)).metadata.schema.column(0).max_definition_level == 0
    _, names = _check(b2, raw, tbl.column_names, bits)
    assert "levels_kernel" not in names, names


def test_dictionary_fallback_is_generated(b2):
    """the fallback writers really switch a chunk from RLE_DICTIONARY to PLAIN pages"""
    tbl, _ = matrix_table(6000, np.random.default_rng(4), "15")
    for w in ("fallback_snappy_1k", "fallback_none_v2"):
        raw = _write(tbl, **WRITERS[w])
        for c in ("i64", "s"):
            enc = [e for k, e in W.page_encodings(raw, 0, tbl.column_names.index(c)) if k != W.DICTIONARY_PAGE]
            first_plain = enc.index(W.PLAIN)
            assert 0 < first_plain and set(enc[:first_plain]) == {W.RLE_DICTIONARY} and set(enc[first_plain:]) == {W.PLAIN}, (w, c, enc)


def test_null_pages_between_full_pages(b2):
    """1 KiB pages: all-valid and all-NULL pages take the uniform short cut and are written by
    fill_uniform_levels_kernel; mixed pages by the level decoder"""
    n = 30000
    rng = np.random.default_rng(8)
    v = rng.integers(0, 100, n)
    mask = ((np.arange(n) // 3000) % 3) == 1
    mask[20000:20010] = True
    tbl = pa.table({"x": pa.array(v, mask=mask), "s": pa.array(["k%d" % x for x in v], mask=mask),
                    "allnull": pa.array([None] * n, pa.int32())})
    for kw in (dict(compression="snappy", data_page_size=1024), dict(compression="none", data_page_size=1024, data_page_version="2.0",
                                                                     use_dictionary=False)):
        raw = _write(tbl, **kw)
        assert pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0).column(0).statistics.null_count == int(mask.sum())
        _, names = _check(b2, raw, ["x", "s", "allnull"])
        assert {"fill_uniform_levels_kernel", "levels_kernel", "expand_nulls_kernel"} <= names, names


DICT_SIZES = [1, 2, 3] + [d for k in (2, 3, 7, 8, 12, 15, 16, 18) for d in (2 ** k, 2 ** k + 1)]


@pytest.mark.parametrize("d", DICT_SIZES)
def test_dictionary_widths(b2, d):
    """dictionaries of d entries: index bit widths 0 to 19, every entry used, 4- and 8-byte, double and string entries"""
    rng = np.random.default_rng(d)
    n = max(4 * d, 4000)
    idx = np.concatenate([rng.permutation(d), rng.integers(0, d, n - d)])
    keys = rng.integers(-2**62, 2**62, d)
    tbl = pa.table({"i32": pa.array(keys[idx].astype(np.int32)), "i64": pa.array(keys[idx]), "f64": pa.array(keys[idx].astype(np.float64)),
                    "s": pa.array(np.array(["s%d" % k for k in keys])[idx])})
    raw = _write(tbl, compression="snappy", dictionary_pagesize_limit=1 << 30, data_page_size=64 << 10)
    for i in range(4):
        assert {e for k, e in W.page_encodings(raw, 0, i) if k != W.DICTIONARY_PAGE} == {W.RLE_DICTIONARY}, i
    _, names = _check(b2, raw, tbl.column_names)
    assert "dict_strings_kernel" in names and "string_chars_kernel" in names, names


def test_snappy_paths_and_in_place_pages(b2):
    """small compressible pages -> snappy_kernel; pages above 192 KiB -> snappy_big_kernel; incompressible pages of
    one snappy literal are read in place: no compressed bytes go through a decompressor"""
    rng = np.random.default_rng(9)
    n = 200_000
    tbl = pa.table({"rep": pa.array(np.repeat(rng.integers(0, 2**40, n // 100), 100)), "noise": pa.array(rng.integers(-2**63, 2**63 - 1, n))})
    for page, kernel in ((8 << 10, "snappy_kernel"), (1 << 20, "snappy_big_kernel")):
        raw = _write(tbl.select(["rep"]), compression="snappy", use_dictionary=False, data_page_size=page, max_rows_per_page=1 << 20)
        _, names = _check(b2, raw, ["rep"])
        assert kernel in names, (page, names)
        assert b2.parquet_last_stats()["compressed_in"] > 0
    schema = pa.schema([pa.field("noise", pa.int64(), nullable=False)])
    raw = _write(tbl.select(["noise"]).cast(schema), compression="snappy", use_dictionary=False, data_page_size=32 << 10)
    _, names = _check(b2, raw, ["noise"])
    st = b2.parquet_last_stats()
    assert st["compressed_in"] == 0 and st["pages"] > 10 and not {"snappy_kernel", "snappy_big_kernel"} & names, (st, names)


def test_timestamps_coerced_to_millis(b2):
    us = pa.array(np.random.default_rng(10).integers(-2**52, 2**52, 5000) * 1000).cast(pa.timestamp("us"))
    raw = _write(pa.table({"t": us}), coerce_timestamps="ms")
    assert "MILLIS" in str(pq.ParquetFile(io.BytesIO(raw)).schema.column(0).logical_type).upper()
    _check(b2, raw, ["t"])


# ---- B. hand-built pages -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_hand_built_pages(b2, name):
    raw, cols, _ = SHAPES[name]()
    _check(b2, raw, cols)


def test_int64_decimal_dtype(b2):
    """INT64 DECIMAL(p <= 9) is DECIMAL32, as INT32 and FIXED_LEN_BYTE_ARRAY decimals of that precision are"""
    for p, dt in ((1, b2.DECIMAL32), (9, b2.DECIMAL32), (10, b2.DECIMAL64), (18, b2.DECIMAL64)):
        raw, cols, _ = W.int64_decimal_shape(p, "plain")
        assert b2.parquet_decode(raw, cols).column(0).dtype == dt, p


# ---- C. malformed input --------------------------------------------------------------------------------------------
def _rejects(b2, raw, cols, code):
    base = b2.device_bytes_in_use()
    with pytest.raises(b2.B2Error) as e:
        b2.parquet_decode(raw, cols)
    assert e.value.code == code, str(e.value)
    assert b2.device_bytes_in_use() == base


def _one_page(col, page, nrows, dict_entries=None, codec=W.UNCOMPRESSED):
    pages = [page]
    if dict_entries is not None:
        pages.insert(0, W.Page(W.DICTIONARY_PAGE, len(dict_entries), W.PLAIN, W.plain(dict_entries, col.ptype)))
    return W.write_file([col], [(nrows, [pages])], codec=codec)


OPT64, REQ64 = W.Column("x", W.INT64, W.OPTIONAL), W.Column("x", W.INT64, W.REQUIRED)


def test_truncated_level_stream_is_rejected(b2):
    """the level stream ends cleanly after 60 of 100 rows: the other 40 rows have no validity.  (This decoded
    "successfully" before, with leftover pool bytes as validity.)  The stream ends at a run boundary, so the level decoder
    reads nothing past the page; the decode raises at the sync after the level pass, before the scan of the validity
    bytes and the NULL expansion, so the 40 unwritten bytes are never read either."""
    for codec in (W.UNCOMPRESSED, W.SNAPPY):
        page = W.Page(W.DATA_PAGE, 100, W.PLAIN, W.def_levels_v1(None, [("rle", 60, 1)]) + W.plain(range(60), W.INT64))
        _rejects(b2, _one_page(OPT64, page, 100, codec=codec), ["x"], ERR_INVALID)
        lv = W.hybrid([("bp", [1] * 8), ("rle", 20, 1)], 1)
        page = W.Page(W.DATA_PAGE_V2, 100, W.PLAIN, W.plain(range(28), W.INT64), levels=lv)
        _rejects(b2, _one_page(OPT64, page, 100, codec=codec), ["x"], ERR_INVALID)


def test_truncated_index_stream_is_rejected(b2):
    """the dictionary index stream ends after 60 of 100 values (REQUIRED), or after 40 of 70 non-NULL values, for INT64
    and STRING columns.  A STRING row the stream does not cover has no source address: the decode raises at the sync
    in front of string_chars_kernel, which would otherwise copy from whatever the unwritten address bytes hold."""
    for col in (REQ64, W.Column("x", W.BYTE_ARRAY, W.REQUIRED, converted=W.CT_UTF8)):
        entries = [5, 6, 7] if col.ptype == W.INT64 else [b"five", b"six", b"seven"]
        page = W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, W.dict_indices([], 2, [("rle", 60, 1)]))
        _rejects(b2, _one_page(col, page, 100, entries), ["x"], ERR_INVALID)
    for col in (OPT64, W.Column("x", W.BYTE_ARRAY, W.OPTIONAL, converted=W.CT_UTF8)):
        entries = [5, 6, 7] if col.ptype == W.INT64 else [b"five", b"six", b"seven"]
        valid = [1] * 70 + [0] * 30
        page = W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, W.def_levels_v1(valid) + W.dict_indices([], 2, [("bp", [1] * 40)]))
        _rejects(b2, _one_page(col, page, 100, entries), ["x"], ERR_INVALID)


def test_string_index_past_the_dictionary_is_rejected(b2):
    """an index past the dictionary leaves its STRING row without a source address, like a truncated stream"""
    col = W.Column("x", W.BYTE_ARRAY, W.REQUIRED, converted=W.CT_UTF8)
    page = W.Page(W.DATA_PAGE, 64, W.RLE_DICTIONARY, W.dict_indices([], 3, [("rle", 32, 1), ("rle", 32, 6)]))
    _rejects(b2, _one_page(col, page, 64, [b"a", b"b", b"c"]), ["x"], ERR_INVALID)


def test_uncompressed_page_sizes_must_agree(b2):
    """an uncompressed page is read in place, so its uncompressed size must be the bytes it holds: one byte less or
    more than compressed_page_size is refused (a larger one would let the decoders read past the page)"""
    for skew in (-1, 1, 1 << 20):
        page = W.Page(W.DATA_PAGE, 100, W.PLAIN, W.plain(range(100), W.INT64), usize_skew=skew)
        _rejects(b2, _one_page(REQ64, page, 100), ["x"], ERR_INVALID)
    good = W.Page(W.DATA_PAGE, 100, W.PLAIN, W.plain(range(100), W.INT64))
    assert b2.parquet_decode(_one_page(REQ64, good, 100), ["x"]).column(0).to_pylist() == list(range(100))


def test_over_claiming_runs_are_rejected(b2):
    """bit-packed runs that announce (far) more values than the page holds, for indexes and for levels, and an RLE run
    whose value bytes are missing"""
    over_idx = W.uvarint((1000 << 1) | 1) + W.bitpack(list(range(16)), 8)
    page = W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, bytes([8]) + over_idx)
    _rejects(b2, _one_page(REQ64, page, 100, list(range(256))), ["x"], ERR_INVALID)
    page = W.Page(W.DATA_PAGE, 1000, W.RLE_DICTIONARY, bytes([8]) + W.uvarint(((1 << 28) << 1) | 1) + b"\x01\x02")
    _rejects(b2, _one_page(REQ64, page, 1000, list(range(256))), ["x"], ERR_INVALID)
    over_lv = W.uvarint((100000 << 1) | 1) + b"\xff\xff"
    page = W.Page(W.DATA_PAGE, 5000, W.PLAIN, struct.pack("<I", len(over_lv)) + over_lv + W.plain(range(16), W.INT64))
    _rejects(b2, _one_page(OPT64, page, 5000), ["x"], ERR_INVALID)
    page = W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, bytes([16]) + W.uvarint(100 << 1) + b"\x01")
    _rejects(b2, _one_page(REQ64, page, 100, [1, 2]), ["x"], ERR_INVALID)


def test_bad_level_length_and_bit_width_are_rejected(b2):
    """a V1 level-length prefix past the page; a page too short for the prefix; levels that consume the page before
    the dictionary bit width; a bit width above 32"""
    body = struct.pack("<I", 1 << 30) + W.hybrid([("rle", 100, 1)], 1) + W.plain(range(100), W.INT64)
    _rejects(b2, _one_page(OPT64, W.Page(W.DATA_PAGE, 100, W.PLAIN, body), 100), ["x"], ERR_INVALID)
    _rejects(b2, _one_page(OPT64, W.Page(W.DATA_PAGE, 100, W.PLAIN, b"\x01\x00"), 100), ["x"], ERR_INVALID)
    _rejects(b2, _one_page(OPT64, W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, W.def_levels_v1([1] * 100)), 100, [1, 2]), ["x"], ERR_INVALID)
    page = W.Page(W.DATA_PAGE, 100, W.RLE_DICTIONARY, bytes([40]) + W.uvarint(100 << 1) + b"\0" * 5)
    _rejects(b2, _one_page(REQ64, page, 100, [1, 2]), ["x"], ERR_INVALID)


def test_short_plain_boolean_page_is_rejected(b2):
    col = W.Column("b", W.BOOLEAN, W.REQUIRED)
    _rejects(b2, _one_page(col, W.Page(W.DATA_PAGE, 1000, W.PLAIN, b"\x55" * 10), 1000), ["b"], ERR_INVALID)
    body = struct.pack("<I", 500) + W.hybrid([("rle", 1000, 1)], 1)
    _rejects(b2, _one_page(col, W.Page(W.DATA_PAGE, 1000, W.RLE, body), 1000), ["b"], ERR_INVALID)


def test_empty_streams_of_all_null_pages_decode(b2):
    """an all-NULL page whose value stream is empty (no bit-width byte, no PLAIN bytes) holds no value to read"""
    col = W.Column("x", W.INT64, W.OPTIONAL)
    pages = [W.Page(W.DICTIONARY_PAGE, 2, W.PLAIN, W.plain([4, 9], W.INT64)),
             W.Page(W.DATA_PAGE, 50, W.RLE_DICTIONARY, W.def_levels_v1([0] * 50)),
             W.Page(W.DATA_PAGE, 10, W.RLE_DICTIONARY, W.def_levels_v1([1] * 10) + W.dict_indices([1] * 10, 1))]
    raw = W.write_file([col], [(60, [pages])])
    _check(b2, raw, ["x"])


@pytest.mark.parametrize("how", ["DELTA_BYTE_ARRAY", "DELTA_LENGTH_BYTE_ARRAY", "BYTE_STREAM_SPLIT", "INT96", "NANOS", "ZSTD"])
def test_unsupported_input_is_refused(b2, how):
    n = 1000
    if how in ("DELTA_BYTE_ARRAY", "DELTA_LENGTH_BYTE_ARRAY"):
        raw = _write(pa.table({"c": pa.array(["v%d" % i for i in range(n)])}), use_dictionary=False, column_encoding={"c": how})
    elif how == "BYTE_STREAM_SPLIT":
        raw = _write(pa.table({"c": pa.array(np.arange(n, dtype=np.float64))}), use_dictionary=False, column_encoding={"c": how})
    elif how == "INT96":
        raw = _write(pa.table({"c": pa.array(np.arange(n)).cast(pa.timestamp("us"))}), use_deprecated_int96_timestamps=True)
    elif how == "NANOS":
        raw = _write(pa.table({"c": pa.array(np.arange(n)).cast(pa.timestamp("ns"))}))
    else:
        raw = _write(pa.table({"c": pa.array(np.arange(n))}), compression="zstd")
    _rejects(b2, raw, ["c"], ERR_UNSUPPORTED)
