"""Exact references for the data-movement layer: gather, slice, concat, the stable partition, the JCUDF row layout and the
shuffle wire format's descriptors.

A column is held as its raw buffers (`Raw`): an (n, width) uint8 matrix for a fixed-width type, Arrow chars + int32 offsets
for STRING, and a bool validity array (None = the column has no validity).  These operations only move bytes, so the
references move the same bytes with numpy indexing and every comparison is bit for bit: NaN payloads, -0.0 and DECIMAL128
included.  Everything is vectorised; oracle/spark_relational.to_rows (one Python loop per row) pins the row layout on small
inputs in tests/test_movement_reference.py.

The helpers that take a module `m` move a Raw to and from the library (like tests/datagen.py's to_b2_*)."""
import ctypes
import struct

import numpy as np

from oracle import spark_cpu as O
from oracle.spark_relational import row_layout  # noqa: F401  (re-exported: the layout the row tests check)

WIDTH = {O.BOOL8: 1, O.INT8: 1, O.INT16: 2, O.INT32: 4, O.INT64: 8, O.FLOAT32: 4, O.FLOAT64: 8, O.DATE32: 4, O.TIMESTAMP_US: 8,
         O.DECIMAL32: 4, O.DECIMAL64: 8, O.DECIMAL128: 16}
# one type of every width, floats for their NaN payloads and -0.0
FIXED_TYPES = [O.INT8, O.BOOL8, O.INT16, O.INT32, O.FLOAT32, O.DATE32, O.INT64, O.FLOAT64, O.TIMESTAMP_US, O.DECIMAL64, O.DECIMAL128]
INT32_MIN = -2**31

# bit patterns worth moving: quiet and signalling NaNs with payloads, -0.0, infinities, integer extremes
_SPECIAL = {
    4: [0x7fc00001, 0xff800001, 0x7f812345, 0x80000000, 0x7f800000, 0xff800000, 0x80000000 - 1, 0x80000000 + 1, 0, 0xffffffff],
    8: [0x7ff8000000000001, 0xfff0000000000001, 0x7ff4000000abcdef, 0x8000000000000000, 0x7ff0000000000000, 0xfff0000000000000,
        0x7fffffffffffffff, 0x8000000000000001, 0, 0xffffffffffffffff],
    16: [(1 << 127), (1 << 127) - 1, (1 << 128) - 1, 1, 0, (1 << 64) - 1, 1 << 64],
    2: [0x8000, 0x7fff, 0xffff, 0],
    1: [0x80, 0x7f, 0xff, 0],
}


class Raw:
    """one column as raw buffers: data (n, width) uint8 | chars uint8 + offsets int32[n + 1]; valid bool[n] or None"""

    def __init__(self, dtype, data=None, valid=None, chars=None, offsets=None, scale=0):
        self.dtype, self.scale = dtype, scale
        self.data, self.chars, self.offsets = data, chars, offsets
        self.valid = None if valid is None else np.asarray(valid, dtype=bool)
        if self.valid is not None and not len(self.valid):
            self.valid = None   # the library gives a zero-row column no validity buffer

    def __len__(self):
        return len(self.offsets) - 1 if self.dtype == O.STRING else len(self.data)

    def valid_or_ones(self):
        return np.ones(len(self), bool) if self.valid is None else self.valid


def rand_fixed(rng, dtype, n, null_frac=0.0, scale=0):
    """random bytes of the type's width, the special patterns of that width at some rows; BOOL8 holds 0 / 1"""
    w = WIDTH[dtype]
    data = rng.integers(0, 256, (n, w), dtype=np.uint8)
    if dtype == O.BOOL8:
        data &= 1
    elif n:
        sp = _SPECIAL[w]
        rows = rng.choice(n, min(n, len(sp)), replace=False)
        for r, v in zip(rows, sp):
            data[r] = np.frombuffer(int(v).to_bytes(w, "little"), np.uint8)
    valid = None if null_frac <= 0 else rng.random(n) >= null_frac
    return Raw(dtype, data=data, valid=valid, scale=scale)


def rand_strings(rng, n, null_frac=0.0, empty_frac=0.2, max_len=40):
    """random byte strings (any byte value), some empty; a NULL row holds no chars"""
    valid = None if null_frac <= 0 else rng.random(n) >= null_frac
    lens = rng.integers(0, max_len + 1, n)
    lens[rng.random(n) < empty_frac] = 0
    if valid is not None:
        lens[~valid] = 0
    offsets = np.zeros(n + 1, np.int32)
    offsets[1:] = np.cumsum(lens)
    return Raw(O.STRING, chars=rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8), offsets=offsets, valid=valid)


def rand_col(rng, dtype, n, null_frac=0.0):
    return rand_strings(rng, n, null_frac) if dtype == O.STRING else rand_fixed(rng, dtype, n, null_frac)


# ---- references ---------------------------------------------------------------------------------------------------------
def _string_take(c, m, keep):
    """chars / offsets of rows m (keep[i] False -> an empty string)"""
    lens = np.where(keep, c.offsets[np.where(keep, m, 0) + 1] - c.offsets[np.where(keep, m, 0)], 0).astype(np.int64)
    offsets = np.zeros(len(m) + 1, np.int64)
    offsets[1:] = np.cumsum(lens)
    total = int(offsets[-1])
    starts = np.where(keep, c.offsets[np.where(keep, m, 0)], 0).astype(np.int64)
    idx = np.repeat(starts - offsets[:-1], lens) + np.arange(total, dtype=np.int64)
    return c.chars[idx], offsets.astype(np.int32)


def gather(c, gmap, nullify_oob):
    """Table.gather of one column: OOB rows (nullify_oob) are NULL with a zero payload / no chars; a NULL row keeps no chars"""
    m = np.asarray(gmap, np.int64)
    n = len(c)
    ok = (m >= 0) & (m < n)
    assert nullify_oob or ok.all(), "without nullify_oob the map must be in range"
    src_valid = c.valid_or_ones()
    valid = ok & src_valid[np.where(ok, m, 0)] if n else np.zeros(len(m), bool)
    out_valid = valid if (nullify_oob or c.valid is not None) else None
    if c.dtype == O.STRING:
        chars, offsets = _string_take(c, m, valid)
        return Raw(O.STRING, chars=chars, offsets=offsets, valid=out_valid)
    data = np.zeros((len(m), WIDTH[c.dtype]), np.uint8)
    data[ok] = c.data[m[ok]]
    return Raw(c.dtype, data=data, valid=out_valid, scale=c.scale)


def take(c, idx):
    return gather(c, idx, False)


def slice_col(c, start, end):
    return take(c, np.arange(start, end))


def concat(parts):
    """Table.concatenate of one column: nullable iff any part is"""
    c0 = parts[0]
    valid = None if all(p.valid is None for p in parts) else np.concatenate([p.valid_or_ones() for p in parts])
    if c0.dtype == O.STRING:
        offs, base = [np.zeros(1, np.int64)], 0
        for p in parts:
            offs.append(p.offsets[1:].astype(np.int64) - p.offsets[0] + base)
            base += int(p.offsets[-1] - p.offsets[0])
        chars = np.concatenate([p.chars[p.offsets[0]:p.offsets[-1]] for p in parts])
        return Raw(O.STRING, chars=chars, offsets=np.concatenate(offs).astype(np.int32), valid=valid)
    return Raw(c0.dtype, data=np.concatenate([p.data for p in parts]), valid=valid, scale=c0.scale)


def stable_partition(pids, nparts):
    """Table.partition: (row order, offsets[nparts + 1]) of a stable counting sort by partition id"""
    pids = np.asarray(pids, np.int64)
    assert ((pids >= 0) & (pids < nparts)).all()
    order = np.argsort(pids, kind="stable")
    offsets = np.zeros(nparts + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(pids, minlength=nparts))
    return order, [int(x) for x in offsets]


# ---- JCUDF rows ---------------------------------------------------------------------------------------------------------
def rows_per_tile(row_bytes):
    """rows one CTA stages per tile in csrc/rows.cu: 96 KB of shared memory, a multiple of 32, 32..1024"""
    return max(32, min(1024, ((96 * 1024) // row_bytes) & ~31))


def to_rows(cols):
    """-> uint8 [n, row_bytes]: every field's payload at its aligned offset (NULL fields too, as the column holds them),
    ceil(ncols / 8) validity bytes, zero gaps and tail"""
    offs, voff, rb = row_layout([c.dtype for c in cols])
    n = len(cols[0])
    out = np.zeros((n, rb), np.uint8)
    for ci, c in enumerate(cols):
        out[:, offs[ci]:offs[ci] + WIDTH[c.dtype]] = c.data
        out[:, voff + ci // 8] |= (c.valid_or_ones().astype(np.uint8) << (ci % 8))
    return out


def defined_bytes(cols):
    """bool [n, row_bytes]: the bytes of to_rows a NULL does not leave open (all but the payload of NULL fields)"""
    offs, _, rb = row_layout([c.dtype for c in cols])
    n = len(cols[0])
    mask = np.ones((n, rb), bool)
    for ci, c in enumerate(cols):
        mask[:, offs[ci]:offs[ci] + WIDTH[c.dtype]] &= c.valid_or_ones()[:, None]
    return mask


def from_rows(rows, dtypes):
    """the columns a row buffer holds: payload bytes of every field, validity bits"""
    offs, voff, _ = row_layout(dtypes)
    return [Raw(dt, data=np.ascontiguousarray(rows[:, offs[ci]:offs[ci] + WIDTH[dt]]),
                valid=((rows[:, voff + ci // 8] >> (ci % 8)) & 1).astype(bool)) for ci, dt in enumerate(dtypes)]


# ---- the B2T1 wire format (csrc/serialize.cu, oracle/shuffle_format.py) --------------------------------------------------
DESC_FIELDS = {"dtype": (0, "<i"), "scale": (4, "<i"), "null_count": (8, "<q"), "validity_bytes": (16, "<q"), "offsets_bytes": (24, "<q"),
               "data_bytes": (32, "<q")}


def _pad64(n):
    return (n + 63) & ~63


def header(buf):
    """-> (ncols, rows, total_bytes)"""
    _, _, ncols, rows, total = struct.unpack_from("<IHHqq", bytes(buf[:24]), 0)
    return ncols, rows, total


def desc(buf, col):
    ncols, _, _ = header(buf)
    assert 0 <= col < ncols
    return {k: struct.unpack_from(f, bytes(buf[24 + 40 * col:24 + 40 * col + 40]), o)[0] for k, (o, f) in DESC_FIELDS.items()}


def set_desc(buf, col, field, value):
    """overwrite one descriptor field of a serialised table held in a writable uint8 array"""
    o, f = DESC_FIELDS[field]
    buf[24 + 40 * col + o:24 + 40 * col + o + struct.calcsize(f)] = np.frombuffer(struct.pack(f, value), np.uint8)


def set_header(buf, field, value):
    o, f = {"ncols": (6, "<H"), "rows": (8, "<q"), "total_bytes": (16, "<q")}[field]
    buf[o:o + struct.calcsize(f)] = np.frombuffer(struct.pack(f, value), np.uint8)


def buffer_offsets(buf):
    """-> per column {"validity", "offsets", "data"}: byte offset of each buffer, as the descriptors lay them out"""
    ncols, _, _ = header(buf)
    off, out = _pad64(24 + 40 * ncols), []
    for c in range(ncols):
        d = desc(buf, c)
        o = {"validity": off}
        off += _pad64(d["validity_bytes"])
        o["offsets"] = off
        off += _pad64(d["offsets_bytes"])
        o["data"] = off
        off += _pad64(d["data_bytes"])
        out.append(o)
    return out


def raw_of_ocol(oc):
    """an oracle OCol (parse / build of oracle/shuffle_format.py) as raw buffers; NULL payloads as the OCol holds them"""
    dt, _, scale = oc.typ
    n = len(oc.values)
    valid = np.asarray(oc.valid, bool)
    if dt == O.STRING:
        enc = [bytes(v) for v in oc.values]
        offsets = np.zeros(n + 1, np.int32)
        offsets[1:] = np.cumsum([len(e) for e in enc]) if n else []
        return Raw(O.STRING, chars=np.frombuffer(b"".join(enc), np.uint8).copy(), offsets=offsets, valid=valid)
    w = WIDTH[dt]
    if O.is_decimal(dt):
        b = b"".join((int(v) & ((1 << (8 * w)) - 1)).to_bytes(w, "little") for v in oc.values)
        data = np.frombuffer(b, np.uint8).reshape(n, w).copy()
    else:
        data = np.ascontiguousarray(np.asarray(oc.values).astype(O._NP[dt])).view(np.uint8).reshape(n, w)
    return Raw(dt, data=data, valid=valid, scale=scale)


def ocol_of_raw(c):
    """Raw -> oracle OCol (the input of oracle/shuffle_format.build); decimals as Python ints"""
    n = len(c)
    if c.dtype == O.STRING or O.is_decimal(c.dtype):
        vals = np.empty(n, dtype=object)
        if c.dtype == O.STRING:
            vals[:] = [c.chars[c.offsets[i]:c.offsets[i + 1]].tobytes() for i in range(n)]
        else:
            vals[:] = [int.from_bytes(c.data[i].tobytes(), "little", signed=True) for i in range(n)]
    else:
        vals = c.data.view(O._NP[c.dtype]).reshape(n).copy()
    return O.OCol(vals, c.valid_or_ones(), (c.dtype, 0, c.scale))


# ---- moving a Raw to and from the library ----------------------------------------------------------------------------------
def _np_values(c):
    if c.dtype == O.DECIMAL128:
        return np.ascontiguousarray(c.data).view(np.uint64).reshape(len(c), 2)
    return np.ascontiguousarray(c.data).view(O._NP[c.dtype] if c.dtype in O._NP else {O.DECIMAL32: np.int32, O.DECIMAL64: np.int64}[c.dtype]).reshape(len(c))


def to_column(m, c):
    if c.dtype == O.STRING:
        return m.Column.from_string_buffers(c.chars, c.offsets, c.valid)
    return m.Column.from_numpy(_np_values(c), dtype=c.dtype, valid=c.valid, scale=c.scale)


def to_table(m, cols):
    return m.Table.from_columns([to_column(m, c) for c in cols])


def from_column(m, col):
    """the column's buffers as the library holds them; valid is None when the column carries no validity"""
    ci = col.info()
    n = ci.size
    vb = np.zeros(max((n + 7) // 8, 1), np.uint8)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    if ci.dtype == O.STRING:
        offsets = np.zeros(n + 1, np.int32)
        chars = np.zeros(max(ci.data_bytes, 1), np.uint8)
        m.check(m.lib.b2_column_to_host(col.h, ptr(chars), ptr(vb), ptr(offsets)))
        out = Raw(O.STRING, chars=chars[:ci.data_bytes], offsets=offsets)
    else:
        data = np.zeros((n, WIDTH[ci.dtype]), np.uint8)
        m.check(m.lib.b2_column_to_host(col.h, ptr(data), ptr(vb), None))
        out = Raw(ci.dtype, data=data, scale=ci.scale)
    out.valid = np.unpackbits(vb, bitorder="little")[:n].astype(bool) if ci.validity else None
    return out


def from_table(m, t):
    return [from_column(m, t.column(i)) for i in range(t.num_columns)]


def assert_same(got, exp, what="", payload="valid", nullability=True):
    """bit-exact comparison of two Raw columns.  payload="valid": fixed-width bytes only where the row is valid; "all": every
    row.  Strings: offsets and chars compared as buffers.  nullability: got carries validity iff exp does."""
    assert got.dtype == exp.dtype, (what, got.dtype, exp.dtype)
    assert len(got) == len(exp), (what, len(got), len(exp))
    if nullability:
        assert (got.valid is None) == (exp.valid is None), (what, "nullable" if got.valid is not None else "not nullable")
    gv, ev = got.valid_or_ones(), exp.valid_or_ones()
    bad = np.flatnonzero(gv != ev)
    assert not len(bad), "%s: validity differs at rows %s (got %s)" % (what, bad[:10], gv[bad[:10]])
    if exp.dtype == O.STRING:
        assert np.array_equal(got.offsets, exp.offsets), "%s: offsets differ at %s" % (what, np.flatnonzero(got.offsets != exp.offsets)[:10])
        assert np.array_equal(got.chars, exp.chars), "%s: chars differ" % what
        return
    assert got.scale == exp.scale, (what, got.scale, exp.scale)
    rows = slice(None) if payload == "all" else ev
    diff = np.flatnonzero((got.data[rows] != exp.data[rows]).any(axis=1))
    assert not len(diff), "%s: payload differs at %d rows, first %s: got %s expected %s" % (
        what, len(diff), diff[:5], got.data[rows][diff[:3]].tolist(), exp.data[rows][diff[:3]].tolist())
