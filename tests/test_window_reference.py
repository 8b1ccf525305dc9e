"""CPU tests (no GPU): the window-function oracle (oracle/spark_window.py) against hand-computed answers and, on random
integer input, against pandas' groupby cumsum / rank / shift."""
import math

import numpy as np
import pytest

from oracle import spark_window as W


def test_rank_dense_rank_row_number_with_ties():
    part = [(1,)] * 6 + [(2,)] * 2
    order = [(10,), (10,), (20,), (30,), (30,), (40,), (5,), (5,)]
    assert W.evaluate(part, order, W.ROW_NUMBER) == [1, 2, 3, 4, 5, 6, 1, 2]
    assert W.evaluate(part, order, W.RANK) == [1, 1, 3, 4, 4, 6, 1, 1]
    assert W.evaluate(part, order, W.DENSE_RANK) == [1, 1, 2, 3, 3, 4, 1, 1]


def test_null_nan_and_signed_zero_keys_form_one_group():
    part = [(None,), (None,), (math.nan,), (float("nan"),), (-0.0,), (0.0,)]
    order = [(1,)] * 6
    assert W.evaluate(part, order, W.ROW_NUMBER) == [1, 2, 1, 2, 1, 2]


def test_running_sum_rows_and_range_frames_with_peers():
    part = [(1,)] * 5
    order = [(1,), (2,), (2,), (3,), (3,)]
    vals = [1, 2, 3, None, 5]
    assert W.evaluate(part, order, W.SUM, vals, frame=W.ROWS, lower=None, upper=0) == [1, 3, 6, 6, 11]
    assert W.evaluate(part, order, W.SUM, vals, frame=W.RANGE, lower=None, upper=0) == [1, 6, 6, 11, 11]
    assert W.evaluate(part, order, W.SUM, vals, frame=W.ROWS, lower=None, upper=None) == [11] * 5
    assert W.evaluate(part, order, W.COUNT, vals, frame=W.ROWS, lower=-1, upper=1) == [2, 3, 2, 2, 1]
    assert W.evaluate(part, order, W.COUNT_ALL, vals, frame=W.ROWS, lower=1, upper=4) == [4, 3, 2, 1, 0]
    assert W.evaluate(part, order, W.SUM, vals, frame=W.ROWS, lower=-5, upper=-1) == [None, 1, 3, 6, 6]
    assert W.evaluate(part, order, W.MIN, vals, frame=W.ROWS, lower=0, upper=0) == [1, 2, 3, None, 5]


def test_lead_lag_at_partition_edges_with_nulls():
    part = [(1,)] * 3 + [(2,)] * 2
    order = [(i,) for i in range(5)]
    vals = [10, None, 30, 40, 50]
    assert W.evaluate(part, order, W.LEAD, vals, offset=1) == [None, 30, None, 50, None]
    assert W.evaluate(part, order, W.LAG, vals, offset=1, default=-1) == [-1, 10, None, -1, 40]
    assert W.evaluate(part, order, W.LAG, vals, offset=0) == vals
    assert W.evaluate(part, order, W.LEAD, vals, offset=5, default=7) == [7] * 5


def test_decimal_running_overflow_is_sticky_and_total_is_not():
    part = [(1,)] * 4
    order = [(i,) for i in range(4)]
    big = 10 ** 38 - 1
    vals = [big, 1, -2, 1]
    run = W.evaluate(part, order, W.SUM, vals, vtype="decimal", lower=None, upper=0, precision=38)
    assert run == [big, None, None, None]
    total = W.evaluate(part, order, W.SUM, vals, vtype="decimal", lower=None, upper=None, precision=38)
    assert total == [big] * 4


def test_float_min_max_order_nan_greatest():
    part = [(1,)] * 3
    order = [(i,) for i in range(3)]
    vals = [math.nan, -0.0, 1.0]
    mx = W.evaluate(part, order, W.MAX, vals, vtype="float", lower=None, upper=None)
    mn = W.evaluate(part, order, W.MIN, vals, vtype="float", lower=None, upper=None)
    assert all(math.isnan(v) for v in mx) and mn == [0.0] * 3


def test_integer_sum_wraps_like_java():
    part = [(1,)] * 2
    order = [(0,), (1,)]
    assert W.evaluate(part, order, W.SUM, [2**63 - 1, 1]) == [2**63 - 1, -2**63]


def test_random_integers_match_pandas():
    pd = pytest.importorskip("pandas")
    rng = np.random.default_rng(3)
    n = 400
    p = np.sort(rng.integers(0, 12, n))
    o = np.zeros(n, dtype=np.int64)
    for g in np.unique(p):   # sorted by (p, o)
        idx = np.nonzero(p == g)[0]
        o[idx] = np.sort(rng.integers(0, 8, len(idx)))
    v = rng.integers(-100, 100, n)
    part, order, vals = [(int(x),) for x in p], [(int(x),) for x in o], [int(x) for x in v]
    df = pd.DataFrame({"p": p, "o": o, "v": v})
    assert W.evaluate(part, order, W.SUM, vals, lower=None, upper=0) == df.groupby("p")["v"].cumsum().tolist()
    assert W.evaluate(part, order, W.RANK) == df.groupby("p")["o"].rank(method="min").astype(int).tolist()
    assert W.evaluate(part, order, W.DENSE_RANK) == df.groupby("p")["o"].rank(method="dense").astype(int).tolist()
    lag = df.groupby("p")["v"].shift(2)
    assert W.evaluate(part, order, W.LAG, vals, offset=2) == [None if np.isnan(x) else int(x) for x in lag]
