"""a6-a9, a11, a12 parity: hash partition (Spark Murmur3), hash join + gather, radix sort / top-N /
bounds / merge, row conversion, concat / slice — CUDA path vs oracle, bit-exact."""
import numpy as np
import pytest

from oracle import spark_cpu as O
from oracle import spark_hash as H
from oracle import spark_relational as R
from tests import datagen as G

pytestmark = pytest.mark.gpu

ALL_KEY_TYPES = [(O.BOOL8, 0, 0), (O.INT8, 0, 0), (O.INT16, 0, 0), (O.INT32, 0, 0), (O.INT64, 0, 0), (O.FLOAT32, 0, 0), (O.FLOAT64, 0, 0),
                 (O.DATE32, 0, 0), (O.TIMESTAMP_US, 0, 0), (O.DECIMAL32, 8, 2), (O.DECIMAL64, 12, 2), (O.DECIMAL128, 30, 4), (O.STRING, 0, 0)]


def gen(rng, typ, n, **kw):
    if typ[0] == O.TIMESTAMP_US:
        c = G.gen_column(rng, (O.INT64, 0, 0), n, **kw)
        return O.OCol(c.values, c.valid, typ)
    return G.gen_column(rng, typ, n, **kw)


# ---- a9 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ALL_KEY_TYPES)
def test_murmur3_per_type(b2, typ):
    rng = np.random.default_rng(typ[0] + 100)
    c = gen(rng, typ, 3000)
    got, _ = b2.murmur3(G.to_b2_table(b2, [c]), [0], 42).to_numpy()
    assert np.array_equal(got, H.murmur3_rows([c], 42))


def test_murmur3_known_answers(b2):
    """Spark: SELECT hash(1), hash(1L) -> -559580957, -1712319331"""
    t = b2.Table.from_columns([b2.Column.from_numpy(np.array([1], np.int32)), b2.Column.from_numpy(np.array([1], np.int64))])
    assert b2.murmur3(t, [0], 42).to_pylist() == [-559580957]
    assert b2.murmur3(t, [1], 42).to_pylist() == [-1712319331]


def test_murmur3_chained_columns_and_seed(b2):
    rng = np.random.default_rng(7)
    cols = [gen(rng, t, 2000) for t in [(O.INT64, 0, 0), (O.STRING, 0, 0), (O.DATE32, 0, 0), (O.DECIMAL128, 38, 6)]]
    t = G.to_b2_table(b2, cols)
    for seed in (42, 107, 114):  # 107 + 7*depth is the agg repartition seed (GpuAggregateExec.scala:219)
        got, _ = b2.murmur3(t, [0, 1, 2, 3], seed).to_numpy()
        assert np.array_equal(got, H.murmur3_rows(cols, seed))


@pytest.mark.parametrize("nparts", [1, 2, 8, 200, 1000])
@pytest.mark.parametrize("n", [0, 1, 5000])
def test_hash_partition(b2, nparts, n):
    rng = np.random.default_rng(nparts + n)
    cols = [gen(rng, (O.INT64, 0, 0), n), gen(rng, (O.STRING, 0, 0), n), gen(rng, (O.DECIMAL64, 12, 2), n)]
    out, offs = b2.hash_partition(G.to_b2_table(b2, cols), [0], nparts)
    exp, eoffs = H.hash_partition(cols, [0], nparts)
    assert offs == eoffs
    for i in range(3):
        G.assert_col_equal(out.column(i), exp[i])


def test_partition_slices_like_reference_suite(b2):
    """GpuPartitioningSuite.scala:112-225: partition indices {0,2,2} over 10 rows -> slices of 2, 0, 8 rows"""
    c = O.OCol(np.arange(10, dtype=np.int32), np.ones(10, bool), (O.INT32, 0, 0))
    t = G.to_b2_table(b2, [c])
    pids = b2.Column.from_numpy(np.array([0, 0] + [2] * 8, np.int32))
    out, offs = b2.partition_by_ids(t, pids, 3)
    assert offs == [0, 2, 2, 10]
    sizes = [b2.slice_table(out, offs[i], offs[i + 1]).num_rows for i in range(3)]
    assert sizes == [2, 0, 8]


# ---- a6/a7 ---------------------------------------------------------------------------------------
def _check_join(b2, build, probe, kind, nulls_equal=False):
    bt, pt = G.to_b2_table(b2, build), G.to_b2_table(b2, probe)
    ht = b2.JoinHashTable(bt, nulls_equal)
    lm, rm = ht.probe(pt, kind)
    elm, erm = R.hash_join(build, probe, kind, nulls_equal)
    glm = lm.to_pylist()
    if rm is None:
        assert erm is None
        assert glm == elm  # semi/anti: stream order
    else:
        grm = rm.to_pylist()
        assert sorted(zip(glm, grm)) == sorted(zip(elm, erm))
        # (output order is unspecified: docs/compatibility.md:18-25; the distinct-build fast path appends per warp)


@pytest.mark.parametrize("kind", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("typ", ALL_KEY_TYPES + [(O.DECIMAL128, 30, 2)])
def test_join_single_key(b2, kind, typ):
    rng = np.random.default_rng(kind * 10 + typ[0])
    nb, ns = (300, 700) if typ[0] == O.BOOL8 else (3000, 7000)     # two BOOL8 keys: every build row matches half the stream
    build = [gen(rng, typ, nb, distinct=800)]
    probe = [gen(rng, typ, ns, distinct=1200)]
    _check_join(b2, build, probe, kind)


def test_join_multi_key_nulls_equal(b2):
    rng = np.random.default_rng(3)
    build = [gen(rng, (O.INT32, 0, 0), 2000, distinct=40, null_frac=0.2), gen(rng, (O.INT64, 0, 0), 2000, distinct=30, null_frac=0.2)]
    probe = [gen(rng, (O.INT32, 0, 0), 3000, distinct=40, null_frac=0.2), gen(rng, (O.INT64, 0, 0), 3000, distinct=30, null_frac=0.2)]
    for ne in (False, True):
        for kind in (0, 1, 2, 3):
            _check_join(b2, build, probe, kind, ne)


def test_join_nulls_equal_packed_keys_nullable_probe(b2):
    """<=> join whose build side has no NULLs (packed 8-byte key regime) probed with NULL keys: a NULL probe key must
    match nothing, whatever bytes sit under the null (GpuHashJoin.scala:602-640)"""
    rng = np.random.default_rng(31)
    build = [gen(rng, (O.INT32, 0, 0), 1500, distinct=40, null_frac=0), gen(rng, (O.INT32, 0, 0), 1500, distinct=5, null_frac=0)]
    probe = [gen(rng, (O.INT32, 0, 0), 3000, distinct=40, null_frac=0.3), gen(rng, (O.INT32, 0, 0), 3000, distinct=5, null_frac=0.3)]
    for col in probe:   # the bytes under a NULL equal a real build key
        col.values[~col.valid] = build[0].values[0]
    for kind in (0, 1, 2, 3, 4):
        _check_join(b2, build, probe, kind, True)
    uniq = [O.OCol(np.arange(500, dtype=np.int64), np.ones(500, bool), (O.INT64, 0, 0))]   # distinct build side: single-pass probe
    pr = [gen(rng, (O.INT64, 0, 0), 3000, distinct=700, null_frac=0.3)]
    pr[0].values[~pr[0].valid] = 7
    for kind in (0, 1, 2, 3, 4):
        _check_join(b2, uniq, pr, kind, True)


def test_join_empty_sides(b2):
    rng = np.random.default_rng(4)
    some, none = [gen(rng, (O.INT64, 0, 0), 100, distinct=10)], [gen(rng, (O.INT64, 0, 0), 0)]
    for kind in (0, 1, 2, 3):
        _check_join(b2, none, some, kind)
        _check_join(b2, some, none, kind)


def test_join_then_gather_payload(b2):
    """q3 shape: orders (build, unique key) JOIN lineitem (stream) then gather payload columns of both sides"""
    rng = np.random.default_rng(5)
    nb, ns = 4000, 20000
    okey = O.OCol(rng.permutation(nb * 4)[:nb].astype(np.int64), np.ones(nb, bool), (O.INT64, 0, 0))
    odate = gen(rng, (O.DATE32, 0, 0), nb, null_frac=0)
    lkey = O.OCol(rng.integers(0, nb * 4, ns).astype(np.int64), np.ones(ns, bool), (O.INT64, 0, 0))
    lprice = gen(rng, (O.DECIMAL64, 12, 2), ns)
    lcomment = gen(rng, (O.STRING, 0, 0), ns)
    ht = b2.JoinHashTable(G.to_b2_table(b2, [okey]))
    lm, rm = ht.probe(G.to_b2_table(b2, [lkey]), 0)
    left = b2.gather(G.to_b2_table(b2, [lkey, lprice, lcomment]), lm)
    right = b2.gather(G.to_b2_table(b2, [okey, odate]), rm)
    elm, erm = R.hash_join([okey], [lkey], 0)
    eleft, eright = R.gather([lkey, lprice, lcomment], elm, False), R.gather([okey, odate], erm, False)
    got = list(zip(*(left.to_pylists() + right.to_pylists())))
    exp = O.rows_of(eleft + eright)
    assert G.norm_rows(got) == G.norm_rows(exp)


def test_gather_nullify_oob(b2):
    rng = np.random.default_rng(6)
    cols = [gen(rng, (O.INT64, 0, 0), 100), gen(rng, (O.STRING, 0, 0), 100), gen(rng, (O.DECIMAL128, 30, 2), 100)]
    gmap = np.array([0, 99, R.INT32_MIN, 5, -1, 100, 7], np.int32)
    out = b2.gather(G.to_b2_table(b2, cols), b2.Column.from_numpy(gmap), True)
    exp = R.gather(cols, gmap, True)
    for i in range(3):
        G.assert_col_equal(out.column(i), exp[i])


# ---- a8 ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ALL_KEY_TYPES)
@pytest.mark.parametrize("asc,nf", [(1, 1), (1, 0), (0, 0), (0, 1)])
@pytest.mark.parametrize("path", ["one-CTA bitonic (n <= 16384)", "radix"])
def test_sort_single_key(b2, typ, asc, nf, path, monkeypatch):
    if path == "radix":
        monkeypatch.setenv("B2_SORT_NO_SMALL", "1")
    else:
        monkeypatch.delenv("B2_SORT_NO_SMALL", raising=False)
    rng = np.random.default_rng(typ[0] * 4 + asc * 2 + nf)
    n = 3000
    k = gen(rng, typ, n, distinct=None if typ[0] in (O.BOOL8,) else 500)
    if typ[0] in (O.FLOAT32, O.FLOAT64):
        k.values[rng.choice(n, 50, replace=False)] = np.nan
        k.values[rng.choice(n, 50, replace=False)] = -0.0
        k.values[rng.choice(n, 50, replace=False)] = 0.0
    payload = O.OCol(np.arange(n, dtype=np.int64), np.ones(n, bool), (O.INT64, 0, 0))
    t = G.to_b2_table(b2, [k, payload])
    perm = b2.sort_order(t, [(0, asc, nf)]).to_pylist()
    assert perm == R.sort_order([k, payload], [(0, asc, nf)])  # stable => unique answer
    out = b2.order_by(t, [(0, asc, nf)])
    exp = R.take([k, payload], perm)
    G.assert_col_equal(out.column(1), exp[1])


def test_sort_multi_key_q3_order(b2):
    """q3: ORDER BY revenue DESC, o_orderdate ASC  (DESC => nulls last, ASC => nulls first)"""
    rng = np.random.default_rng(11)
    n = 20000
    rev = gen(rng, (O.DECIMAL128, 36, 4), n, distinct=300)
    date = gen(rng, (O.DATE32, 0, 0), n, distinct=50)
    key = O.OCol(np.arange(n, dtype=np.int64), np.ones(n, bool), (O.INT64, 0, 0))
    cols = [rev, date, key]
    keys = [(0, 0, 0), (1, 1, 1)]
    t = G.to_b2_table(b2, cols)
    assert b2.sort_order(t, keys).to_pylist() == R.sort_order(cols, keys)
    # the one-CTA bitonic sort of small inputs (multi-chunk keys, duplicates, non-power-of-two sizes): same stable order
    for m in (2, 3, 1000, 8191, 8192, 8193, 16384):
        sub = [O.OCol(c.values[:m], c.valid[:m], c.typ) for c in cols]
        assert b2.sort_order(G.to_b2_table(b2, sub), keys).to_pylist() == R.sort_order(sub, keys)
    top = b2.top_n(t, keys, 10)
    exp = R.take(cols, R.sort_order(cols, keys)[:10])
    for i in range(3):
        G.assert_col_equal(top.column(i), exp[i])


@pytest.mark.parametrize("n", [0, 1, 2, 4097, 100000])
def test_sort_sizes_and_sortedness(b2, n):
    rng = np.random.default_rng(n)
    vals = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    t = b2.Table.from_columns([b2.Column.from_numpy(vals)])
    got, _ = b2.order_by(t, [(0, 1, 1)]).column(0).to_numpy()
    assert np.array_equal(got, np.sort(vals))


def test_merge_and_bounds(b2):
    rng = np.random.default_rng(12)
    a = np.sort(rng.integers(0, 1000, 500)).astype(np.int64)
    b = np.sort(rng.integers(0, 1000, 700)).astype(np.int64)
    ta, tb = b2.Table.from_columns([b2.Column.from_numpy(a)]), b2.Table.from_columns([b2.Column.from_numpy(b)])
    merged, _ = b2.merge_sorted([ta, tb], [(0, 1, 1)]).column(0).to_numpy()
    assert np.array_equal(merged, np.sort(np.concatenate([a, b])))
    probe = rng.integers(-5, 1005, 300).astype(np.int64)
    tp = b2.Table.from_columns([b2.Column.from_numpy(probe)])
    lo, _ = b2.search_bounds(ta, tp, [(0, 1, 1)], False).to_numpy()
    hi, _ = b2.search_bounds(ta, tp, [(0, 1, 1)], True).to_numpy()
    assert np.array_equal(lo, np.searchsorted(a, probe, "left"))
    assert np.array_equal(hi, np.searchsorted(a, probe, "right"))


# ---- a11 / a12 -----------------------------------------------------------------------------------
def test_rows_roundtrip_and_layout(b2):
    rng = np.random.default_rng(13)
    types = [(O.INT8, 0, 0), (O.INT64, 0, 0), (O.INT16, 0, 0), (O.DECIMAL128, 30, 2), (O.INT32, 0, 0), (O.FLOAT64, 0, 0), (O.BOOL8, 0, 0),
             (O.DATE32, 0, 0), (O.DECIMAL64, 12, 2)]
    n = 3000
    cols = [gen(rng, t, n, small=(t[0] in (O.FLOAT64,))) for t in types]
    for c in cols:  # nulls carry zero payload in the oracle rows; make the inputs agree
        if c.values.dtype == object:
            c.values[~c.valid] = 0
        else:
            c.values[~c.valid] = 0
    t = G.to_b2_table(b2, cols)
    rows = b2.table_to_rows(t)
    exp = R.to_rows(cols)
    assert rows.shape == exp.shape
    assert np.array_equal(rows, exp)
    back = b2.table_from_rows(rows, [c.typ[0] for c in cols], [c.typ[2] for c in cols])
    for i, c in enumerate(cols):
        G.assert_col_equal(back.column(i), c)


def test_concat_and_slice(b2):
    rng = np.random.default_rng(14)
    types = [(O.INT64, 0, 0), (O.STRING, 0, 0), (O.DECIMAL128, 30, 2), (O.BOOL8, 0, 0)]
    parts = [[gen(rng, t, n, null_frac=nf) for t in types] for n, nf in [(100, 0.2), (0, 0.0), (37, 0.0), (2500, 0.5)]]
    out = b2.concat([G.to_b2_table(b2, p) for p in parts])
    for i, t in enumerate(types):
        exp = O.OCol(np.concatenate([p[i].values for p in parts]), np.concatenate([p[i].valid for p in parts]), t)
        G.assert_col_equal(out.column(i), exp)
        sl = b2.slice_table(out, 90, 150).column(i)
        G.assert_col_equal(sl, O.OCol(exp.values[90:150], exp.valid[90:150], t))


def test_full_outer_join_then_gather(b2):
    """FullOuter: every stream row and every build row appears; the unmatched side is NULL after the gather with
    out-of-bounds -> NULL (JoinGatherer.scala:585-599); distinct and duplicate build keys, NULL keys on both sides"""
    rng = np.random.default_rng(21)
    for distinct in (True, False):
        bkey = gen(rng, (O.INT64, 0, 0), 4000, distinct=4000 if distinct else 500)
        pkey = gen(rng, (O.INT64, 0, 0), 9000, distinct=3000)
        bval = gen(rng, (O.DECIMAL64, 12, 2), 4000)
        ht = b2.JoinHashTable(G.to_b2_table(b2, [bkey]))
        lm, rm = ht.probe(G.to_b2_table(b2, [pkey]), 4)
        elm, erm = R.hash_join([bkey], [pkey], 4)
        assert sorted(zip(lm.to_pylist(), rm.to_pylist())) == sorted(zip(elm, erm))
        left = b2.gather(G.to_b2_table(b2, [pkey]), lm, True)
        right = b2.gather(G.to_b2_table(b2, [bkey, bval]), rm, True)
        order = np.lexsort((rm.to_numpy()[0], lm.to_numpy()[0]))
        eorder = np.lexsort((np.array(erm), np.array(elm)))
        el = R.gather([pkey], np.array(elm)[eorder], True)
        er = R.gather([bkey, bval], np.array(erm)[eorder], True)
        gl = b2.gather(left, b2.Column.from_numpy(order.astype(np.int32)))
        gr = b2.gather(right, b2.Column.from_numpy(order.astype(np.int32)))
        G.assert_col_equal(gl.column(0), el[0])
        G.assert_col_equal(gr.column(0), er[0])
        G.assert_col_equal(gr.column(1), er[1])


def test_join_probe_through_selection_vector(b2):
    """late materialisation: filter row ids + probe through them == filter, then probe; the left map holds ORIGINAL row ids"""
    import ctypes
    rng = np.random.default_rng(41)
    nb, ns = 3000, 20000
    build = [gen(rng, (O.INT64, 0, 0), nb, distinct=4000, null_frac=0.02)]
    key = gen(rng, (O.INT64, 0, 0), ns, distinct=5000, null_frac=0.05)
    flt = gen(rng, (O.INT32, 0, 0), ns, distinct=10, null_frac=0.1)
    st = G.to_b2_table(b2, [key, flt])
    pred = G.b2_expr_col(b2, 1, flt) < b2.lit(4, b2.INT32)
    prog = b2.Program([pred])
    ids = ctypes.c_int64()
    b2.check(b2.lib.b2_filter_row_ids(prog.h, st.h, ctypes.byref(ids)))
    sel = b2.Column(ids.value)
    keep = O.eval_expr(pred.sexpr, [key, flt])
    mask = keep.valid & (keep.values != 0)
    assert sel.to_pylist() == [int(i) for i in np.flatnonzero(mask)]
    ht = b2.JoinHashTable(G.to_b2_table(b2, build))
    keys_only = b2.Table.from_columns([st.column(0)])
    for kind in (0, 1, 2, 3):
        lm, rm = ctypes.c_int64(), ctypes.c_int64()
        b2.check(b2.lib.b2_join_probe_sel(ht.h, keys_only.h, sel.h, kind, ctypes.byref(lm), ctypes.byref(rm)))
        glm = b2.Column(lm.value).to_pylist()
        grm = b2.Column(rm.value).to_pylist() if rm.value else None
        fkey = O.OCol(key.values[mask], key.valid[mask], key.typ)
        elm, erm = R.hash_join(build, [fkey], kind)
        orig = np.flatnonzero(mask)
        elm = [int(orig[i]) for i in elm]
        if grm is None:
            assert glm == elm
        else:
            assert sorted(zip(glm, grm)) == sorted(zip(elm, erm))


@pytest.mark.parametrize("n", [65536, 65536 + 1, 200_003, 1_000_000 + 15])
def test_simple_predicate_row_ids_fast_path(b2, n, monkeypatch):
    """conjunctions of NOT NULL integer column vs literal comparisons take the specialised kernel (simplefilter.cu); its row ids
    equal the VM's and the numpy restatement for every width, every comparison and a ragged last tile"""
    import ctypes
    rng = np.random.default_rng(n)
    cols = {
        "i8": (rng.integers(-100, 100, n).astype(np.int8), b2.INT8),
        "i16": (rng.integers(-3000, 3000, n).astype(np.int16), b2.INT16),
        "i32": (rng.integers(-2**31, 2**31 - 1, n).astype(np.int32), b2.INT32),
        "i64": (rng.integers(-2**62, 2**62, n).astype(np.int64), b2.INT64),
        "date": (rng.integers(8000, 11000, n).astype(np.int32), b2.DATE32),
    }
    names = list(cols)
    t = b2.Table.from_columns([b2.Column.from_numpy(cols[k][0], dtype=cols[k][1]) if cols[k][1] == b2.DATE32 else b2.Column.from_numpy(cols[k][0]) for k in names])
    c = {k: b2.col(i, cols[k][1], nullable=False) for i, k in enumerate(names)}
    v = {k: cols[k][0] for k in names}
    cases = [
        (c["date"] < b2.lit(9204, b2.DATE32), v["date"] < 9204),
        ((c["date"] >= b2.lit(8500, b2.DATE32)) & (c["date"] < b2.lit(10000, b2.DATE32)) & (c["i8"] > b2.lit(-5, b2.INT8)) & (c["i16"] != b2.lit(7, b2.INT16)),
         (v["date"] >= 8500) & (v["date"] < 10000) & (v["i8"] > -5) & (v["i16"] != 7)),
        ((c["i64"] <= b2.lit(1 << 40, b2.INT64)) & (c["i32"] > b2.lit(-12345, b2.INT32)), (v["i64"] <= (1 << 40)) & (v["i32"] > -12345)),
        ((c["i8"] == b2.lit(3, b2.INT8)) & (c["i64"] >= b2.lit(-(1 << 61), b2.INT64)), (v["i8"] == 3) & (v["i64"] >= -(1 << 61))),
        (c["i32"] > b2.lit(2**31 - 1, b2.INT32), np.zeros(n, bool)),
    ]
    for pred, mask in cases:
        prog = b2.Program([pred])
        got = []
        for env in (None, "1"):
            if env: monkeypatch.setenv("B2_FILTER_NO_SIMPLE", env)
            else: monkeypatch.delenv("B2_FILTER_NO_SIMPLE", raising=False)
            ids = ctypes.c_int64()
            b2.check(b2.lib.b2_filter_row_ids(prog.h, t.h, ctypes.byref(ids)))
            got.append(b2.Column(ids.value).to_numpy()[0])
        want = np.flatnonzero(mask).astype(np.int32)
        assert np.array_equal(got[0], want) and np.array_equal(got[1], want)
    monkeypatch.delenv("B2_FILTER_NO_SIMPLE", raising=False)
