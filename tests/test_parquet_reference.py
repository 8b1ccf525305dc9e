"""CPU tests (no GPU): the hand-built Parquet writer of tests/parquet_pages.py.  pyarrow must read every shape the GPU
tests decode back to the values the builder meant, and the RLE / bit-packed hybrid encoder must round-trip through an
independent small decoder, so that a GPU mismatch can only be the GPU's."""
import io
import struct

import numpy as np
import pyarrow.parquet as pq
import pytest

from oracle import spark_cpu as O
from oracle import spark_parquet as P
from tests import parquet_pages as W

SHAPES = W.all_shapes()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_pyarrow_reads_what_the_builder_meant(name):
    raw, cols, expect = SHAPES[name]()
    for c, oc in zip(cols, P.read_parquet(raw, cols)):
        got = [v if ok else None for v, ok in zip(oc.values, oc.valid)]
        assert len(got) == len(expect[c]), (c, len(got), len(expect[c]))
        bad = [(i, g, e) for i, (g, e) in enumerate(zip(got, expect[c])) if (g is None) != (e is None) or (g is not None and g != e)]
        assert not bad, (c, bad[:5])


def test_int64_decimal_is_decimal32_up_to_precision_9():
    """the expected dtype of an INT64 DECIMAL(p <= 9) is DECIMAL32 (the oracle maps by precision, as Spark does)"""
    for p, dt in ((1, O.DECIMAL32), (9, O.DECIMAL32), (10, O.DECIMAL64), (18, O.DECIMAL64)):
        raw, cols, _ = W.int64_decimal_shape(p, "delta")
        assert pq.ParquetFile(io.BytesIO(raw)).metadata.schema.column(0).physical_type == "INT64"
        assert P.read_parquet(raw, cols)[0].typ[0] == dt


def test_dictionary_payload_alignment():
    """dict_alignment_shape(r) really puts each dictionary payload at r (mod 8)"""
    for r in range(8):
        raw, cols, _ = W.dict_alignment_shape(r)
        md = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0)
        for i in range(len(cols)):
            off = md.column(i).dictionary_page_offset
            hdr_len = len(W.Page(W.DICTIONARY_PAGE, 300, W.PLAIN, b"\0" * {0: 1200, 1: 2400, 2: 2400}[i]).encode(W.UNCOMPRESSED)[0])
            assert (off + hdr_len) % 8 == r


def test_v2_pages_declare_their_compression():
    raw, _, _ = W.v2_mixed_compression_shape()
    md = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(0)
    assert md.column(0).compression == "SNAPPY" and md.column(1).compression == "SNAPPY"


def test_thrift_compact_known_bytes():
    """field headers (short delta form and long form), zigzag varints, lists, nested structs and booleans, from the
    Thrift compact protocol specification"""
    assert W.Compact.struct([(1, "i32", 3)]) == b"\x15\x06\x00"
    assert W.Compact.struct([(1, "i32", -1), (2, "i64", 150)]) == b"\x15\x01\x16\xac\x02\x00"
    assert W.Compact.struct([(20, "i32", 1)]) == b"\x05\x28\x02\x00"
    assert W.Compact.struct([(3, "bool", True), (4, "bool", False)]) == b"\x31\x12\x00"
    assert W.Compact.struct([(1, "list", ("i32", [1, 2]))]) == b"\x19\x25\x02\x04\x00"
    assert W.Compact.struct([(1, "list", ("i32", list(range(15))))])[:3] == b"\x19\xf5\x0f"
    assert W.Compact.struct([(2, "struct", [(1, "binary", "ab")])]) == b"\x2c\x18\x02ab\x00\x00"
    assert W.uvarint(300) == b"\xac\x02"


def test_hybrid_known_bytes():
    """the example of the Parquet specification (Encodings.md): 0..7 at bit width 3 is 0x88 0xC6 0xFA"""
    assert W.bitpack(list(range(8)), 3) == b"\x88\xc6\xfa"
    assert W.hybrid([("bp", list(range(8)))], 3) == b"\x03\x88\xc6\xfa"
    assert W.hybrid([("rle", 5, 0x1234)], 13) == b"\x0a\x34\x12"


@pytest.mark.parametrize("bw", list(range(1, 33)))
def test_hybrid_roundtrip_every_width(bw):
    rng = np.random.default_rng(bw)
    vals = [int(v) for v in rng.integers(0, 1 << bw, 700, dtype=np.uint64)]
    vals[100:140] = [vals[100]] * 40
    vals[300:301] = [(1 << bw) - 1]
    runs = W.auto_runs(vals)
    assert any(r[0] == "rle" for r in runs) and any(r[0] == "bp" for r in runs)
    assert W.HybridDecoder.decode(W.hybrid(runs, bw), bw, len(vals)) == vals


@pytest.mark.parametrize("length", list(range(1, 10)) + [127, 128, 129, 1000])
def test_hybrid_roundtrip_run_lengths(length):
    vals = [5] * length
    assert W.HybridDecoder.decode(W.hybrid([("rle", length, 5)], 4), 4, length) == vals
    tail = [(3 * k) % 16 for k in range(length)]
    for pad in (0, 15):
        enc = W.hybrid([("rle", 3, 1), ("bp", tail, pad)], 4)
        assert W.HybridDecoder.decode(enc, 4, 3 + length) == [1, 1, 1] + tail
    # a bit-packed run in the middle carries whole groups: its padding decodes to values
    mid = W.hybrid([("bp", tail, 15), ("rle", 2, 9)], 4)
    assert W.HybridDecoder.decode(mid, 4, len(tail) + (-len(tail) % 8) + 2)[len(tail):] == [15] * (-len(tail) % 8) + [9, 9]


def test_hybrid_decoder_rejects_truncation():
    enc = W.hybrid([("rle", 10, 1), ("bp", list(range(8)))], 3)
    with pytest.raises(ValueError):
        W.HybridDecoder.decode(enc, 3, 19)
    with pytest.raises(ValueError):
        W.HybridDecoder.decode(enc[:-1], 3, 18)
    assert W.HybridDecoder.decode(W.bp_run([1, 0, 1], 1, groups=1), 1, 3) == [1, 0, 1]


def test_levels_v1_prefix():
    body = W.def_levels_v1([1, 1, 0, 1])
    (n,) = struct.unpack("<I", body[:4])
    assert n == len(body) - 4 and W.HybridDecoder.decode(body[4:], 1, 4) == [1, 1, 0, 1]


def test_page_encodings_reader():
    """the page-header reader the GPU tests use to prove a dictionary fallback sees each page of a built chunk"""
    raw, _, _ = W.v2_mixed_compression_shape()
    assert W.page_encodings(raw, 0, 0) == [(W.DICTIONARY_PAGE, W.PLAIN)] + [(W.DATA_PAGE_V2, W.RLE_DICTIONARY)] * 8
    assert W.page_encodings(raw, 0, 1) == [(W.DATA_PAGE_V2, W.PLAIN)] * 8


def test_delta_binary_packed_pages_are_what_pyarrow_reads():
    """the DELTA_BINARY_PACKED encoder: wrapping 64-bit deltas, a partial last block, one value, zero-width miniblocks"""
    import pyarrow as pa
    rng = np.random.default_rng(5)
    for vals in ([7], [3] * 300, [int(x) for x in rng.integers(-2**63, 2**63 - 1, 1000, endpoint=True)],
                 [int(x) for x in np.cumsum(rng.integers(-5, 50, 517))]):
        col = W.Column("x", W.INT64, W.REQUIRED)
        raw = W.write_file([col], [(len(vals), [[W.Page(W.DATA_PAGE, len(vals), W.DELTA_BINARY_PACKED, W.delta_binary_packed(vals))]])])
        assert W.page_encodings(raw, 0, 0) == [(W.DATA_PAGE, W.DELTA_BINARY_PACKED)]
        assert pq.read_table(pa.BufferReader(raw)).column(0).to_pylist() == vals

