"""The data-movement references (tests/movement_reference.py) against the oracle's row-at-a-time restatements and against
hand-computed cases.  CPU only."""
import numpy as np
import pytest

from oracle import shuffle_format as F
from oracle import spark_cpu as O
from oracle import spark_hash as H
from oracle import spark_relational as R
from tests import movement_reference as M


def _ocol(c):
    return M.ocol_of_raw(c)


@pytest.mark.parametrize("dtypes", [
    [O.INT8, O.INT64, O.INT16, O.DECIMAL128, O.INT32, O.FLOAT64, O.BOOL8, O.DATE32, O.DECIMAL64],
    [O.DECIMAL128],
    [O.INT8] * 17,
    [O.BOOL8, O.DECIMAL128, O.INT16, O.FLOAT32, O.TIMESTAMP_US, O.INT8, O.DECIMAL32, O.INT64],
])
def test_to_rows_matches_the_row_at_a_time_oracle(dtypes):
    rng = np.random.default_rng(len(dtypes))
    n = 37
    cols = [M.rand_fixed(rng, dt, n, null_frac=0.3) for dt in dtypes]
    for c in cols:   # struct.pack of a Python float does not keep every NaN payload: keep the oracle's floats finite
        if c.dtype in (O.FLOAT32, O.FLOAT64):
            c.data[:] = np.frombuffer(rng.standard_normal(n).astype(O._NP[c.dtype]).tobytes(), np.uint8).reshape(n, -1)
    assert np.array_equal(M.to_rows(cols), R.to_rows([_ocol(c) for c in cols]))
    back = M.from_rows(M.to_rows(cols), dtypes)
    for c, b in zip(cols, back):
        assert np.array_equal(b.data, c.data) and np.array_equal(b.valid, c.valid)


def test_defined_bytes_leave_only_null_payloads_open():
    rng = np.random.default_rng(1)
    dtypes = [O.INT8, O.INT64, O.DECIMAL128, O.INT16]   # offsets 0, 8, 16, 32; validity at 34; 40-byte rows
    cols = [M.rand_fixed(rng, dt, 50, null_frac=0.4) for dt in dtypes]
    assert R.row_layout(dtypes) == ([0, 8, 16, 32], 34, 40)
    mask = M.defined_bytes(cols)
    open_bytes = sum(int((~c.valid).sum()) * M.WIDTH[c.dtype] for c in cols)
    assert int((~mask).sum()) == open_bytes
    assert mask[:, 1:8].all() and mask[:, 34:].all()   # the gap after the INT8 and the validity byte + tail


def test_rows_per_tile_range():
    assert M.rows_per_tile(8) == 1024 and M.rows_per_tile(96) == 1024 and M.rows_per_tile(104) == 928
    assert M.rows_per_tile(64 * 16 + 8) == 64
    assert M.rows_per_tile(520) == 160


@pytest.mark.parametrize("nullify", [False, True])
@pytest.mark.parametrize("dtype", [O.INT32, O.DECIMAL128, O.STRING])
def test_gather_matches_the_oracle(dtype, nullify):
    rng = np.random.default_rng(dtype)
    c = M.rand_col(rng, dtype, 40, null_frac=0.3)
    gmap = rng.integers(-3 if nullify else 0, 43 if nullify else 40, 60)
    if nullify:
        gmap[:3] = [M.INT32_MIN, 40, 39]
    got = M.gather(c, gmap, nullify)
    exp = R.gather([_ocol(c)], gmap, nullify)[0]
    assert got.valid.tolist() == exp.valid.tolist()
    assert _ocol(got).to_pylist() == exp.to_pylist()
    if dtype != O.STRING:   # OOB rows: zero payload; an in-range NULL row keeps the bytes under it
        oob = (gmap < 0) | (gmap >= 40)
        assert not got.data[oob].any()
        assert np.array_equal(got.data[~oob], c.data[gmap[~oob]])
    else:
        lens = np.diff(got.offsets)
        assert not lens[~got.valid].any()


def test_gather_keeps_nullability():
    rng = np.random.default_rng(2)
    c = M.rand_fixed(rng, O.INT64, 10)
    assert M.gather(c, [1, 2], False).valid is None
    assert M.gather(c, [1, 2], True).valid.all()
    assert M.gather(c, [], True).valid is None   # a zero-row column carries no validity
    s = M.rand_strings(rng, 10)
    assert M.gather(s, [3, 3, 0], False).valid is None


def test_string_take_row_by_row():
    rng = np.random.default_rng(3)
    s = M.rand_strings(rng, 200, null_frac=0.2)
    idx = rng.integers(0, 200, 500)
    got = M.take(s, idx)
    words = [s.chars[s.offsets[i]:s.offsets[i + 1]].tobytes() for i in range(200)]
    assert [got.chars[got.offsets[i]:got.offsets[i + 1]].tobytes() for i in range(500)] == [words[i] for i in idx]
    assert got.offsets[0] == 0 and got.offsets[-1] == len(got.chars)


def test_concat_and_slice_rebase_strings():
    rng = np.random.default_rng(4)
    s = M.rand_strings(rng, 30, null_frac=0.2)
    a, b = M.slice_col(s, 3, 11), M.slice_col(s, 11, 30)
    assert a.offsets[0] == 0 and b.offsets[0] == 0
    whole = M.concat([a, M.slice_col(s, 5, 5), b])
    assert np.array_equal(whole.offsets, s.offsets[3:] - s.offsets[3])
    assert np.array_equal(whole.chars, s.chars[s.offsets[3]:])
    x, y = M.rand_fixed(rng, O.INT16, 5), M.rand_fixed(rng, O.INT16, 7, null_frac=0.5)
    xy = M.concat([x, y])
    assert xy.valid is not None and xy.valid[:5].all() and np.array_equal(xy.valid[5:], y.valid)
    assert M.concat([x, x]).valid is None


def test_stable_partition_matches_the_hash_oracle():
    rng = np.random.default_rng(5)
    keys = [O.OCol(rng.integers(0, 50, 300).astype(np.int64), np.ones(300, bool), (O.INT64, 0, 0))]
    for nparts in (1, 3, 7):
        pids = H.partition_ids(keys, nparts)
        order, offs = M.stable_partition(pids, nparts)
        exp, eoffs = H.hash_partition(keys, [0], nparts)
        assert offs == eoffs and keys[0].values[order].tolist() == exp[0].values.tolist()
        for p in range(nparts):   # stable: row ids rise inside a partition
            assert np.all(np.diff(order[offs[p]:offs[p + 1]]) > 0)
    order, offs = M.stable_partition([2, 0, 2, 1, 0], 4)
    assert order.tolist() == [1, 4, 3, 0, 2] and offs == [0, 2, 3, 5, 5]


def test_wire_helpers_follow_the_oracle_writer():
    rng = np.random.default_rng(6)
    cols = [M.rand_fixed(rng, O.INT32, 70, null_frac=0.3), M.rand_strings(rng, 70, null_frac=0.2), M.rand_fixed(rng, O.DECIMAL128, 70)]
    buf = np.frombuffer(F.build([M.ocol_of_raw(c) for c in cols]), np.uint8).copy()
    assert M.header(buf) == (3, 70, len(buf))
    d = M.desc(buf, 1)
    assert d["dtype"] == O.STRING and d["offsets_bytes"] == 71 * 4 and d["data_bytes"] == int(cols[1].offsets[-1])
    offs = M.buffer_offsets(buf)
    assert np.array_equal(np.frombuffer(buf, np.int32, 71, offs[1]["offsets"]), cols[1].offsets)
    assert np.array_equal(np.unpackbits(buf[offs[0]["validity"]:offs[0]["validity"] + 9], bitorder="little")[:70].astype(bool), cols[0].valid)
    assert np.array_equal(buf[offs[2]["data"]:offs[2]["data"] + 70 * 16].reshape(70, 16), cols[2].data)
    M.set_desc(buf, 0, "null_count", 5)
    assert M.desc(buf, 0)["null_count"] == 5
    M.set_header(buf, "rows", 3)
    assert M.header(buf)[1] == 3
    parsed = F.parse(F.build([M.ocol_of_raw(c) for c in cols]))
    for c, p in zip(cols, parsed):
        M.assert_same(M.raw_of_ocol(p), c, payload="valid", nullability=False)
