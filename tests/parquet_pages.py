"""A minimal Parquet writer for tests: pages and files whose every byte the test chooses, written from the Apache Parquet
format specification (parquet.thrift, Encodings.md) and the Thrift compact protocol specification.

pyarrow never writes some of the shapes the GPU decoder has separate code for: dictionary indexes declared wider than
needed, hundreds of short runs per page, RLE runs longer than the page, garbage in the padding of the last bit-packed
group, bit-packed definition levels, BOOLEAN as RLE in V1 pages, INT64 decimals of precision <= 9, uncompressed V2 pages
inside a snappy chunk, dictionary pages at any file alignment.  This module builds them; pyarrow reading the same bytes
is the expected value (tests/test_parquet_reference.py checks that it reads what the builder meant).

Layers: `Compact` (Thrift compact encoder), `hybrid` / `HybridDecoder` (RLE / bit-packed hybrid), `plain` (PLAIN
values), `Page` (one page: header fields + body), `Column` (schema element) and `write_file` (PAR1, chunks, footer)."""
import struct

import numpy as np
import pyarrow as pa

# parquet.thrift enums
BOOLEAN, INT32, INT64, INT96, FLOAT, DOUBLE, BYTE_ARRAY, FLBA = range(8)
REQUIRED, OPTIONAL = 0, 1
PLAIN, PLAIN_DICTIONARY, RLE, BIT_PACKED, DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY, RLE_DICTIONARY, \
    BYTE_STREAM_SPLIT = 0, 2, 3, 4, 5, 6, 7, 8, 9
UNCOMPRESSED, SNAPPY = 0, 1
DATA_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 2, 3
CT_UTF8, CT_DECIMAL, CT_DATE, CT_TIMESTAMP_MILLIS, CT_TIMESTAMP_MICROS, CT_INT_8, CT_INT_16 = 0, 5, 6, 9, 10, 15, 16


def uvarint(n):
    assert n >= 0
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def zigzag(n):
    return (n << 1) ^ (n >> 63)


class Compact:
    """Thrift compact protocol writer.  A struct is a list of (field id, type, value); type is one of the names below,
    `struct` values are such lists again, `list` values are (element type, [elements])."""
    TYPES = {"bool": None, "i32": 5, "i64": 6, "binary": 8, "list": 9, "struct": 12}

    @classmethod
    def struct(cls, fields):
        out, last = bytearray(), 0
        for fid, typ, val in fields:
            if val is None:
                continue
            code = (1 if val else 2) if typ == "bool" else cls.TYPES[typ]
            delta = fid - last
            out += bytes([(delta << 4) | code]) if 0 < delta <= 15 else bytes([code]) + uvarint(zigzag(fid))
            last = fid
            if typ != "bool":
                out += cls.value(typ, val)
        out.append(0)
        return bytes(out)

    @classmethod
    def value(cls, typ, val):
        if typ in ("i32", "i64"):
            return uvarint(zigzag(val) & ((1 << 64) - 1))
        if typ == "binary":
            val = val.encode() if isinstance(val, str) else val
            return uvarint(len(val)) + val
        if typ == "struct":
            return cls.struct(val)
        if typ == "list":
            et, items = val
            n = len(items)
            head = bytes([(n << 4) | cls.TYPES[et]]) if n < 15 else bytes([0xF0 | cls.TYPES[et]]) + uvarint(n)
            return head + b"".join(cls.value(et, v) for v in items)
        raise ValueError(typ)


# ---- RLE / bit-packed hybrid ---------------------------------------------------------------------------------------
def bitpack(values, bw):
    """values (a multiple of 8 of them) packed LSB first, `bw` bits each"""
    assert len(values) % 8 == 0
    acc, nbits, out = 0, 0, bytearray()
    for v in values:
        assert 0 <= v < (1 << bw) or bw == 0
        acc |= int(v) << nbits
        nbits += bw
        while nbits >= 8:
            out.append(acc & 0xFF)
            acc >>= 8
            nbits -= 8
    assert nbits == 0
    return bytes(out)


def rle_run(count, value, bw):
    return uvarint(count << 1) + int(value).to_bytes((bw + 7) // 8, "little")


def bp_run(values, bw, pad=0, groups=None):
    """bit-packed run of `values`, the last group filled with `pad`; `groups` overrides the count in the header"""
    vals = list(values) + [pad] * (-len(values) % 8)
    g = len(vals) // 8
    return uvarint(((g if groups is None else groups) << 1) | 1) + bitpack(vals, bw)


def hybrid(runs, bw):
    """runs: ("rle", count, value) | ("bp", values) | ("bp", values, pad) -> the encoded stream"""
    out = bytearray()
    for r in runs:
        out += rle_run(r[1], r[2], bw) if r[0] == "rle" else bp_run(r[1], bw, *r[2:])
    return bytes(out)


def auto_runs(values, min_rle=8):
    """runs for `values`: RLE for repeats of at least `min_rle`, bit-packed groups of 8 between them.  The last
    bit-packed run may be padded; since it ends the stream the padding decodes to no value."""
    values = list(values)
    runs, i, lit = [], 0, []
    while i < len(values):
        j = i
        while j < len(values) and values[j] == values[i]:
            j += 1
        if j - i >= min_rle and len(lit) % 8 == 0:
            if lit:
                runs.append(("bp", lit))
                lit = []
            runs.append(("rle", j - i, values[i]))
            i = j
        else:
            lit.append(values[i])
            i += 1
    if lit:
        runs.append(("bp", lit))
    return runs


class HybridDecoder:
    """decodes `count` values of a hybrid stream; raises ValueError when the stream ends early"""

    @staticmethod
    def decode(buf, bw, count):
        out, pos = [], 0
        while len(out) < count:
            if pos >= len(buf):
                raise ValueError("stream ends after %d of %d values" % (len(out), count))
            h, shift = 0, 0
            while True:
                b = buf[pos]
                pos += 1
                h |= (b & 0x7F) << shift
                shift += 7
                if not b & 0x80:
                    break
            if h & 1:
                n = (h >> 1) * 8
                nbytes = n * bw // 8
                if pos + nbytes > len(buf):
                    raise ValueError("bit-packed run past the stream")
                acc = int.from_bytes(buf[pos:pos + nbytes], "little")
                out += [(acc >> (k * bw)) & ((1 << bw) - 1) for k in range(n)]
                pos += nbytes
            else:
                vb = (bw + 7) // 8
                if pos + vb > len(buf) or h >> 1 == 0:
                    raise ValueError("bad RLE run")
                out += [int.from_bytes(buf[pos:pos + vb], "little")] * (h >> 1)
                pos += vb
        return out[:count]


# ---- values ----------------------------------------------------------------------------------------------------------
def plain(values, ptype, type_length=0):
    """PLAIN encoding of non-NULL values (ints, floats, bools, bytes; FLBA: big-endian two's complement ints)"""
    if ptype == BOOLEAN:
        bits = [1 if v else 0 for v in values]
        bits += [0] * (-len(bits) % 8)
        return bitpack(bits, 1)
    if ptype == INT32:
        return np.asarray(values, dtype=np.int64).astype(np.int32).tobytes()
    if ptype == INT64:
        return np.asarray(values).astype(np.int64).tobytes()
    if ptype == FLOAT:
        return np.asarray(values, dtype=np.float32).tobytes()
    if ptype == DOUBLE:
        return np.asarray(values, dtype=np.float64).tobytes()
    if ptype == BYTE_ARRAY:
        return b"".join(struct.pack("<I", len(v)) + v for v in values)
    if ptype == FLBA:
        return b"".join(int(v).to_bytes(type_length, "big", signed=True) for v in values)
    raise ValueError(ptype)


def delta_binary_packed(values, block=128, miniblocks=4):
    """DELTA_BINARY_PACKED (Encodings.md) of 64-bit values: header (block size, miniblocks per block, value count,
    zigzag first value), then per block the zigzag minimum delta, one bit width per miniblock and the miniblocks
    bit-packed LSB first.  Deltas wrap modulo 2^64; the last block is padded with zero (relative) deltas."""
    m64 = (1 << 64) - 1
    vals = [int(v) & m64 for v in values]
    out = bytearray(uvarint(block) + uvarint(miniblocks) + uvarint(len(vals)))
    first = vals[0] - (1 << 64) if vals and vals[0] >> 63 else (vals[0] if vals else 0)
    out += uvarint(zigzag(first) & m64)
    signed = lambda d: d - (1 << 64) if d >> 63 else d
    deltas = [signed((b - a) & m64) for a, b in zip(vals, vals[1:])]
    per = block // miniblocks
    for s0 in range(0, len(deltas), block):
        blk = deltas[s0:s0 + block]
        md = min(blk)
        rel = [(d - md) & m64 for d in blk] + [0] * (block - len(blk))
        widths = [max(x.bit_length() for x in rel[k * per:(k + 1) * per]) for k in range(miniblocks)]
        out += uvarint(zigzag(md) & m64) + bytes(widths)
        for k in range(miniblocks):
            out += bitpack(rel[k * per:(k + 1) * per], widths[k]) if widths[k] else b""
    return bytes(out)


def def_levels_v1(valid, runs=None):
    """V1 definition levels of a flat OPTIONAL column: 4-byte length + hybrid stream at bit width 1"""
    body = hybrid(runs if runs is not None else auto_runs([int(v) for v in valid]), 1)
    return struct.pack("<I", len(body)) + body


def dict_indices(idx, bw, runs=None):
    """RLE_DICTIONARY data: bit-width byte + hybrid stream of the indexes"""
    return bytes([bw]) + hybrid(runs if runs is not None else auto_runs(idx), bw)


# ---- pages, chunks, files -------------------------------------------------------------------------------------------
class Page:
    """kind: DATA_PAGE / DATA_PAGE_V2 / DICTIONARY_PAGE.  `body`: the uncompressed payload (V1: levels + values; V2:
    values only, levels in `levels`).  `compress` (V2 pages of a snappy chunk): is_compressed."""

    def __init__(self, kind, num_values, encoding, body, levels=b"", num_nulls=0, compress=True, usize_skew=0):
        self.kind, self.num_values, self.encoding, self.body = kind, num_values, encoding, body
        self.levels, self.num_nulls, self.compress, self.usize_skew = levels, num_nulls, compress, usize_skew

    def encode(self, codec):
        squeeze = codec == SNAPPY and (self.kind != DATA_PAGE_V2 or self.compress)
        payload = pa.compress(self.body, codec="snappy", asbytes=True) if squeeze else self.body
        usize, csize = len(self.levels) + len(self.body) + self.usize_skew, len(self.levels) + len(payload)
        hdr = [(1, "i32", self.kind), (2, "i32", usize), (3, "i32", csize)]
        if self.kind == DATA_PAGE:
            hdr.append((5, "struct", [(1, "i32", self.num_values), (2, "i32", self.encoding), (3, "i32", RLE), (4, "i32", RLE)]))
        elif self.kind == DICTIONARY_PAGE:
            hdr.append((7, "struct", [(1, "i32", self.num_values), (2, "i32", PLAIN)]))
        else:
            hdr.append((8, "struct", [(1, "i32", self.num_values), (2, "i32", self.num_nulls), (3, "i32", self.num_values),
                                      (4, "i32", self.encoding), (5, "i32", len(self.levels)), (6, "i32", 0),
                                      (7, "bool", bool(self.compress))]))
        return Compact.struct(hdr), self.levels + payload, usize


class Column:
    def __init__(self, name, ptype, repetition=OPTIONAL, converted=None, scale=None, precision=None, type_length=None):
        self.name, self.ptype, self.repetition = name, ptype, repetition
        self.converted, self.scale, self.precision, self.type_length = converted, scale, precision, type_length

    def schema(self):
        return [(1, "i32", self.ptype), (2, "i32", self.type_length), (3, "i32", self.repetition), (4, "binary", self.name),
                (6, "i32", self.converted), (7, "i32", self.scale), (8, "i32", self.precision)]


def write_file(columns, row_groups, codec=UNCOMPRESSED, dict_payload_align=None):
    """columns: [Column]; row_groups: [(num_rows, [[Page] per column])] -> the file's bytes.  A dictionary page is
    written first in its chunk.  dict_payload_align = (m, r): filler bytes in front of each chunk that has a
    dictionary page put that page's payload at a file offset = r (mod m)."""
    out = bytearray(b"PAR1")
    rgs = []
    for nrows, chunks in row_groups:
        metas = []
        for col, pages in zip(columns, chunks):
            encoded = [p.encode(codec) for p in pages]
            has_dict = bool(pages) and pages[0].kind == DICTIONARY_PAGE
            if has_dict and dict_payload_align:
                m, r = dict_payload_align
                out += b"\xee" * ((r - (len(out) + len(encoded[0][0]))) % m)
            start = len(out)
            for hdr, payload, _ in encoded:
                out += hdr + payload
            data_off = start + (len(encoded[0][0]) + len(encoded[0][1]) if has_dict else 0)
            nvals = sum(p.num_values for p in pages if p.kind != DICTIONARY_PAGE)
            encs = sorted({p.encoding for p in pages} | {RLE})
            md = [(1, "i32", col.ptype), (2, "list", ("i32", encs)), (3, "list", ("binary", [col.name])), (4, "i32", codec),
                  (5, "i64", nvals), (6, "i64", sum(len(h) + u for h, _, u in encoded)), (7, "i64", len(out) - start),
                  (9, "i64", data_off), (11, "i64", start if has_dict else None)]
            metas.append((start, md, len(out) - start))
        rgs.append([(1, "list", ("struct", [[(2, "i64", s), (3, "struct", md)] for s, md, _ in metas])),
                    (2, "i64", sum(n for _, _, n in metas)), (3, "i64", nrows)])
    schema = [[(4, "binary", "schema"), (5, "i32", len(columns))]] + [c.schema() for c in columns]
    footer = Compact.struct([(1, "i32", 1), (2, "list", ("struct", schema)), (3, "i64", sum(n for n, _ in row_groups)),
                             (4, "list", ("struct", rgs)), (6, "binary", "b2 test writer")])
    return bytes(out + footer + struct.pack("<I", len(footer)) + b"PAR1")



# ---- the shapes the GPU tests decode ---------------------------------------------------------------------------------
# Each shape is (file bytes, column names, expected columns); an expected column is a list of python values with None
# for NULL: ints (decimals unscaled), floats, bools, bytes.

def _levels(valid, runs=None):
    return def_levels_v1(valid, runs)


def _dict_chunk(col, entries, idx, valid, bw, nvals_per_page, kind=DATA_PAGE, runs_of=None, compress=True):
    """dictionary page + RLE_DICTIONARY data pages of `nvals_per_page` rows; `runs_of(page_idx_values)` picks the runs"""
    pages = [Page(DICTIONARY_PAGE, len(entries), PLAIN, plain(entries, col.ptype, col.type_length or 0))]
    for s in range(0, len(idx), nvals_per_page):
        v = valid[s:s + nvals_per_page]
        dense = [int(i) for i, ok in zip(idx[s:s + nvals_per_page], v) if ok]
        body = dict_indices(dense, bw, runs_of(dense) if runs_of else None)
        if col.repetition == REQUIRED:
            pages.append(Page(kind, len(v), RLE_DICTIONARY, body, compress=compress))
        elif kind == DATA_PAGE:
            pages.append(Page(kind, len(v), RLE_DICTIONARY, _levels(v) + body))
        else:
            lv = hybrid(auto_runs([int(x) for x in v]), 1)
            pages.append(Page(kind, len(v), RLE_DICTIONARY, body, levels=lv, num_nulls=int(len(v) - sum(v)), compress=compress))
    return pages


def _expect(entries, idx, valid):
    return [entries[int(i)] if ok else None for i, ok in zip(idx, valid)]


def _entries(ptype, d, rng, type_length=0):
    if ptype == INT32:
        return [int(x) for x in rng.integers(-2**31, 2**31, d)]
    if ptype == INT64:
        return [int(x) for x in rng.integers(-2**63, 2**63 - 1, d, endpoint=True)]
    if ptype == DOUBLE:
        return [float(x) for x in rng.standard_normal(d) * 1e6]
    if ptype == BYTE_ARRAY:
        return [b"v%d" % i + b"\xc3\xa9" * (i % 3) for i in range(d)]
    if ptype == FLBA:
        lim = 2 ** (8 * type_length - 1)
        return [int(x) % (2 * lim) - lim for x in rng.integers(0, 2**62, d)]
    raise ValueError(ptype)


def dict_width_shape(bw, n=1000):
    """every value type through dictionary indexes declared `bw` bits wide (wider than the dictionary needs from
    bw = 10 on): 4- and 8-byte entries (the put4 fast path), doubles, strings and 6-byte FLBA decimals (the scalar put)"""
    rng = np.random.default_rng(100 + bw)
    d = min(1 << bw, 700)
    cols = [Column("i32", INT32, REQUIRED), Column("i64", INT64, OPTIONAL), Column("f64", DOUBLE, REQUIRED),
            Column("s", BYTE_ARRAY, OPTIONAL, converted=CT_UTF8),
            Column("dec", FLBA, OPTIONAL, converted=CT_DECIMAL, scale=2, precision=14, type_length=6)]
    idx = rng.integers(0, d, n)
    idx[100:260] = d - 1                       # an RLE run of the largest index
    chunks, expect = [], {}
    for c in cols:
        valid = np.ones(n, bool) if c.repetition == REQUIRED else rng.random(n) >= 0.2
        entries = _entries(c.ptype, d, rng, c.type_length or 0)
        chunks.append(_dict_chunk(c, entries, idx, valid, bw, 400))
        expect[c.name] = _expect(entries, idx, valid)
    return write_file(cols, [(n, chunks)]), [c.name for c in cols], expect


def run_count_shape(nruns):
    """one page of `nruns` index runs (alternating 3-value RLE runs and one bit-packed group) and as many level runs"""
    rng = np.random.default_rng(nruns)
    idx_runs, idx = [], []
    for r in range(nruns):
        if r % 2 == 0:
            v = int(rng.integers(0, 50))
            idx_runs.append(("rle", 3, v)); idx += [v] * 3
        else:
            g = [int(x) for x in rng.integers(0, 50, 8)]
            idx_runs.append(("bp", g)); idx += g
    lv_runs, valid = [], []
    while len(valid) < len(idx) + 1000:
        lv_runs.append(("rle", 2, 0)); valid += [0, 0]
        lv_runs.append(("rle", 3, 1)); valid += [1, 1, 1]
    # trim the levels to exactly len(idx) valid rows
    out_valid, k = [], 0
    for v in valid:
        if k == len(idx):
            break
        out_valid.append(v); k += v
    lv_runs = auto_runs(out_valid, min_rle=2)
    entries = _entries(INT64, 50, rng)
    col = Column("x", INT64, OPTIONAL)
    page = Page(DATA_PAGE, len(out_valid), RLE_DICTIONARY, _levels(out_valid, lv_runs) + dict_indices(idx, 6, idx_runs))
    dense = iter(idx)
    expect = [entries[next(dense)] if ok else None for ok in out_valid]
    return write_file([col], [(len(out_valid), [[Page(DICTIONARY_PAGE, 50, PLAIN, plain(entries, INT64)), page]])]), ["x"], {"x": expect}


def run_length_shape(last_bp, pad):
    """RLE runs of 1-9 and 127-129 values and bit-packed runs of 1-17 groups (the 128-value put4 step), ending in a
    bit-packed run of `last_bp` values whose last group is padded with `pad` (which is past the dictionary when 255)"""
    rng = np.random.default_rng(last_bp * 3 + pad)
    runs, idx = [], []
    for length in list(range(1, 10)) + [127, 128, 129]:
        v = int(rng.integers(0, 200))
        runs.append(("rle", length, v)); idx += [v] * length
        g = [int(x) for x in rng.integers(0, 200, 8 * (1 + length % 17))]
        runs.append(("bp", g)); idx += g
    tail = [int(x) for x in rng.integers(0, 200, last_bp)]
    runs.append(("bp", tail, pad)); idx += tail
    cols, chunks, expect = [], [], {}
    for name, ptype in (("i32", INT32), ("i64", INT64), ("s", BYTE_ARRAY)):
        entries = _entries(ptype, 200, rng)
        c = Column(name, ptype, REQUIRED)
        cols.append(c)
        chunks.append([Page(DICTIONARY_PAGE, 200, PLAIN, plain(entries, ptype)), Page(DATA_PAGE, len(idx), RLE_DICTIONARY, dict_indices(idx, 8, runs))])
        expect[name] = [entries[i] for i in idx]
    return write_file(cols, [(len(idx), chunks)]), [c.name for c in cols], expect


def long_rle_shape():
    """RLE runs that announce more values than the page has: the levels (one run of num_values + 100: the uniform-page
    short cut; a bit-packed group then a run past the end) and the indexes"""
    n = 300
    entries = [7, -9, 11]
    col = Column("x", INT64, OPTIONAL)
    p1 = Page(DATA_PAGE, n, RLE_DICTIONARY, _levels([1] * n, [("rle", n + 100, 1)]) + dict_indices([], 2, [("rle", 5000, 2)]))
    lv = [1, 0, 1, 1, 0, 0, 1, 0]
    p2 = Page(DATA_PAGE, n, RLE_DICTIONARY, _levels(lv + [1] * (n - 8), [("bp", lv), ("rle", 1000, 1)])
              + dict_indices([], 2, [("bp", [0, 1, 2, 0, 1, 2, 0, 1]), ("rle", 1 << 20, 1)]))
    dense2 = ([0, 1, 2, 0, 1, 2, 0, 1] + [1] * n)[:sum(lv) + n - 8]
    it = iter(dense2)
    expect = [entries[2]] * n + [entries[next(it)] if ok else None for ok in lv + [1] * (n - 8)]
    pages = [Page(DICTIONARY_PAGE, 3, PLAIN, plain(entries, INT64)), p1, p2]
    return write_file([col], [(2 * n, [pages])]), ["x"], {"x": expect}


def bitpacked_levels_shape(codec):
    """definition levels written only as bit-packed groups (no RLE run at all), last group padded with ones, over PLAIN
    INT32, DOUBLE and BOOLEAN values in V1 pages"""
    rng = np.random.default_rng(7)
    n, per = 2003, 500
    cols = [Column("i", INT32), Column("d", DOUBLE), Column("b", BOOLEAN)]
    chunks, expect = [], {}
    for c in cols:
        valid = rng.random(n) >= 0.3
        valid[1000:1100] = True
        vals = {INT32: lambda: [int(x) for x in rng.integers(-2**31, 2**31, n)], DOUBLE: lambda: [float(x) for x in rng.standard_normal(n)],
                BOOLEAN: lambda: [bool(x) for x in rng.integers(0, 2, n)]}[c.ptype]()
        pages = []
        for s in range(0, n, per):
            v = [int(x) for x in valid[s:s + per]]
            dense = [x for x, ok in zip(vals[s:s + per], v) if ok]
            pages.append(Page(DATA_PAGE, len(v), PLAIN, _levels(v, [("bp", v, 1)]) + plain(dense, c.ptype)))
        chunks.append(pages)
        expect[c.name] = [x if ok else None for x, ok in zip(vals, valid)]
    return write_file(cols, [(n, chunks)], codec=codec), [c.name for c in cols], expect


def int64_decimal_shape(p, encoding):
    """DECIMAL(p, min(p, 2)) stored as INT64 (pyarrow stores p <= 18 as INT64 only with store_decimal_as_integer, and p <= 9
    then as INT32): ±(10^p − 1), 0, ±1 and random values, PLAIN, dictionary or DELTA_BINARY_PACKED encoded, with NULLs"""
    rng = np.random.default_rng(p)
    lim = 10 ** p - 1
    n = 600
    vals = [int(x) % (2 * lim + 1) - lim for x in rng.integers(0, 2**62, n)]
    vals[:5] = [lim, -lim, 0, 1, -1]
    valid = rng.random(n) >= 0.1
    valid[:5] = True
    col = Column("d", INT64, OPTIONAL, converted=CT_DECIMAL, scale=min(p, 2), precision=p)
    if encoding == "dict":
        entries = sorted(set(vals))
        pos = {v: i for i, v in enumerate(entries)}
        idx = [pos[v] for v in vals]
        pages = _dict_chunk(col, entries, idx, valid, max(1, (len(entries) - 1).bit_length()), 250)
    else:
        enc, values = {"plain": (PLAIN, lambda d: plain(d, INT64)), "delta": (DELTA_BINARY_PACKED, delta_binary_packed)}[encoding]
        pages = []
        for s in range(0, n, 250):
            v = valid[s:s + 250]
            pages.append(Page(DATA_PAGE, len(v), enc, _levels(v) + values([x for x, ok in zip(vals[s:s + 250], v) if ok])))
    return write_file([col], [(n, [pages])]), ["d"], {"d": [x if ok else None for x, ok in zip(vals, valid)]}


def v2_mixed_compression_shape():
    """a snappy chunk of V2 pages that alternate is_compressed = true / false, dictionary and PLAIN, with NULLs"""
    rng = np.random.default_rng(22)
    n, per = 4000, 500
    col_d, col_p = Column("d", INT64, OPTIONAL), Column("p", INT32, REQUIRED)
    entries = _entries(INT64, 40, rng)
    idx = rng.integers(0, 40, n)
    valid = rng.random(n) >= 0.25
    dpages = [Page(DICTIONARY_PAGE, 40, PLAIN, plain(entries, INT64))]
    ppages = []
    pv = [int(x) for x in rng.integers(-2**31, 2**31, n)]
    for k, s in enumerate(range(0, n, per)):
        v = [int(x) for x in valid[s:s + per]]
        dense = [int(i) for i, ok in zip(idx[s:s + per], v) if ok]
        dpages.append(Page(DATA_PAGE_V2, len(v), RLE_DICTIONARY, dict_indices(dense, 6), levels=hybrid(auto_runs(v), 1),
                           num_nulls=len(v) - sum(v), compress=k % 2 == 0))
        ppages.append(Page(DATA_PAGE_V2, per, PLAIN, plain(pv[s:s + per], INT32), compress=k % 2 == 1))
    raw = write_file([col_d, col_p], [(n, [dpages, ppages])], codec=SNAPPY)
    return raw, ["d", "p"], {"d": _expect(entries, idx, valid), "p": pv}


def dict_alignment_shape(r):
    """uncompressed dictionary pages (read in place) whose payload starts at file offset = r (mod 8): the put4 fast path
    needs the entries aligned to their width"""
    rng = np.random.default_rng(40 + r)
    cols, chunks, expect = [], [], {}
    n = 1100
    for name, ptype in (("i32", INT32), ("i64", INT64), ("f64", DOUBLE)):
        c = Column(name, ptype, REQUIRED)
        entries = _entries(ptype, 300, rng)
        idx = rng.integers(0, 300, n)
        cols.append(c)
        chunks.append(_dict_chunk(c, entries, idx, np.ones(n, bool), 9, n))
        expect[name] = _expect(entries, idx, np.ones(n, bool))
    return write_file(cols, [(n, chunks)], dict_payload_align=(8, r)), [c.name for c in cols], expect


def boolean_rle_shape(kind):
    """BOOLEAN as RLE (4-byte length + hybrid stream at width 1) in V1 or V2 pages, OPTIONAL, with an all-NULL page"""
    rng = np.random.default_rng(kind)
    n, per = 1500, 300
    vals = [bool(x) for x in rng.integers(0, 2, n)]
    vals[300:450] = [True] * 150
    valid = rng.random(n) >= 0.2
    valid[600:900] = False
    pages = []
    for s in range(0, n, per):
        v = [int(x) for x in valid[s:s + per]]
        dense = [int(x) for x, ok in zip(vals[s:s + per], v) if ok]
        body = hybrid(auto_runs(dense), 1)
        body = struct.pack("<I", len(body)) + body
        if kind == DATA_PAGE:
            pages.append(Page(DATA_PAGE, len(v), RLE, _levels(v) + body))
        else:
            pages.append(Page(DATA_PAGE_V2, len(v), RLE, body, levels=hybrid(auto_runs(v), 1), num_nulls=len(v) - sum(v)))
    raw = write_file([Column("b", BOOLEAN)], [(n, [pages])])
    return raw, ["b"], {"b": [x if ok else None for x, ok in zip(vals, valid)]}


def all_shapes():
    """name -> builder; every shape tests/test_parquet_paths_gpu.py decodes"""
    out = {"dict_bw%d" % bw: (lambda bw=bw: dict_width_shape(bw)) for bw in range(1, 33)}
    out.update({"runs%d" % k: (lambda k=k: run_count_shape(k)) for k in (65, 129, 1001)})
    out.update({"run_lengths_%d_pad%d" % (m, pad): (lambda m=m, pad=pad: run_length_shape(m, pad))
                for m in (1, 7, 8, 9, 96, 97, 127, 128, 129, 200) for pad in (0, 255)})
    out["long_rle"] = long_rle_shape
    out.update({"bitpacked_levels_%s" % c: (lambda c=c: bitpacked_levels_shape(c)) for c in (UNCOMPRESSED, SNAPPY)})
    out.update({"int64_decimal_p%d_%s" % (p, d): (lambda p=p, d=d: int64_decimal_shape(p, d))
                for p in (1, 5, 9, 10, 18) for d in ("plain", "dict", "delta")})
    out["v2_mixed_compression"] = v2_mixed_compression_shape
    out.update({"dict_align%d" % r: (lambda r=r: dict_alignment_shape(r)) for r in range(8)})
    out.update({"boolean_rle_v%d" % (1 if k == DATA_PAGE else 2): (lambda k=k: boolean_rle_shape(k)) for k in (DATA_PAGE, DATA_PAGE_V2)})
    return out


def page_encodings(raw, row_group, column):
    """[(page type, encoding)] of one column chunk, from its page headers (Thrift compact reader for PageHeader)"""
    import io
    import pyarrow.parquet as pq
    md = pq.ParquetFile(io.BytesIO(raw)).metadata.row_group(row_group).column(column)
    pos = md.dictionary_page_offset if md.has_dictionary_page else md.data_page_offset
    end, out = pos + md.total_compressed_size, []

    def varint():
        nonlocal pos
        v, sh = 0, 0
        while True:
            b = raw[pos]
            pos += 1
            v |= (b & 0x7F) << sh
            sh += 7
            if not b & 0x80:
                return v

    def read_struct(depth):
        nonlocal pos
        fields, last = {}, 0
        while True:
            b = raw[pos]
            pos += 1
            if b == 0:
                return fields
            typ, delta = b & 0x0F, b >> 4
            fid = last + delta if delta else (lambda z: (z >> 1) ^ -(z & 1))(varint())
            last = fid
            if typ in (1, 2):
                fields[fid] = typ == 1
            elif typ in (3,):
                pos += 1
            elif typ in (4, 5, 6):
                z = varint()
                fields[fid] = (z >> 1) ^ -(z & 1)
            elif typ == 8:
                n = varint()
                pos += n
            elif typ == 12:
                fields[fid] = read_struct(depth + 1)
            else:
                raise ValueError("thrift type %d in a page header" % typ)

    while pos < end:
        h = read_struct(0)
        kind = h[1]
        sub = h.get(5) or h.get(7) or h.get(8) or {}
        out.append((kind, sub.get(4 if kind == DATA_PAGE_V2 else 2)))
        pos += h[3]
    return out
