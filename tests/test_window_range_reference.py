"""CPU tests (no GPU): the RANGE-by-value oracle (tests/window_range_oracle.py) against hand-computed frames, against the RANGE
frames of oracle/spark_window.py that its (UNBOUNDED, 0) and (UNBOUNDED, UNBOUNDED) frames stand for, and against pandas'
time-based rolling windows."""
import numpy as np
import pytest

from oracle import spark_window as W
from tests import window_range_oracle as R

P7 = [(1,)] * 7
V7 = [1, 2, 3, 4, 5, 6, 7]


def test_ascending_nulls_first_with_ties():
    order = [(None,), (None,), (1,), (2,), (2,), (5,), (9,)]
    # the NULL rows' frame is their peer group; a non-NULL row's frame holds no NULL row
    assert R.evaluate(P7, order, W.SUM, V7, lower=-1, upper=0) == [3, 3, 3, 12, 12, 6, 7]
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=1, upper=3) == [2, 2, 2, 1, 1, 0, 0]
    assert R.evaluate(P7, order, W.SUM, V7, lower=1, upper=3) == [3, 3, 9, 6, 6, None, None]
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=-3, upper=-1) == [2, 2, 0, 1, 1, 2, 0]
    assert R.evaluate(P7, order, W.MIN, V7, lower=0, upper=0) == [1, 1, 3, 4, 4, 6, 7]
    # UNBOUNDED PRECEDING holds the leading NULLs of nulls first
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=None, upper=1) == [2, 2, 5, 5, 5, 6, 7]
    assert R.evaluate(P7, order, W.MAX, V7, lower=0, upper=None) == [7] * 7


def test_descending_nulls_last():
    order = [(9,), (5,), (2,), (2,), (1,), (None,), (None,)]
    kw = dict(ascending=False, nulls_first=False)
    # DESC negates the offsets: 1 PRECEDING reaches the values up to v + 1
    assert R.evaluate(P7, order, W.SUM, V7, lower=-1, upper=0, **kw) == [1, 2, 7, 7, 12, 13, 13]
    # UNBOUNDED FOLLOWING holds the trailing NULLs of nulls last
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=-1, upper=None, **kw) == [7, 6, 5, 5, 5, 2, 2]
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=None, upper=1, **kw) == [1, 2, 5, 5, 5, 7, 7]
    assert R.evaluate(P7, order, W.COUNT_ALL, V7, lower=1, upper=4, **kw) == [1, 3, 1, 1, 0, 2, 2]


def test_partitions_bound_the_frame():
    part = [(1,)] * 3 + [(2,)] * 3
    order = [(1,), (2,), (3,), (1,), (2,), (3,)]
    vals = [1, 10, 100, 1000, 10000, 100000]
    assert R.evaluate(part, order, W.SUM, vals, lower=-5, upper=5) == [111] * 3 + [111000] * 3
    assert R.evaluate(part, order, W.SUM, vals, lower=-1, upper=1) == [11, 111, 110, 11000, 111000, 110000]


def test_bounds_past_the_type_range_do_not_wrap():
    part = [(1,)] * 3
    i8 = [(-128,), (0,), (127,)]
    assert R.evaluate(part, i8, W.COUNT_ALL, lower=-300, upper=300) == [3, 3, 3]
    assert R.evaluate(part, i8, W.COUNT_ALL, lower=1, upper=300) == [2, 1, 0]
    assert R.evaluate(part, i8, W.COUNT_ALL, lower=-127, upper=127) == [1, 2, 2]
    big = 2 ** 63 - 2
    i64 = [(-2 ** 63,), (-2 ** 63 + 2,), (2 ** 63 - 1,)]
    # 2^63 - 1 + big wraps to a negative upper bound value in 64 bits
    assert R.evaluate(part, i64, W.COUNT_ALL, lower=-big, upper=big) == [2, 2, 1]
    assert R.evaluate(part, i64[::-1], W.COUNT_ALL, lower=-big, upper=big, ascending=False) == [1, 2, 2]
    assert R.evaluate(part, i64, W.COUNT_ALL, lower=big, upper=big) == [0, 0, 0]
    d38 = [(-(10 ** 38 - 1),), (0,), (10 ** 38 - 1,)]
    assert R.evaluate(part, d38, W.COUNT_ALL, lower=-big, upper=big) == [1, 1, 1]


def test_decimal_sum_is_null_only_when_the_frame_total_does_not_fit():
    part = [(1,)] * 4
    order = [(i,) for i in range(4)]
    big = 10 ** 38 - 1
    vals = [big, 1, -2, 1]
    got = R.evaluate(part, order, W.SUM, vals, vtype="decimal", lower=-1, upper=0, precision=38)
    assert got == [big, None, -1, -1]
    # the (UNBOUNDED, 0) alias keeps the sticky running rule
    assert R.evaluate(part, order, W.SUM, vals, vtype="decimal", lower=None, upper=0, precision=38) == [big, None, None, None]


@pytest.mark.parametrize("lower,upper", [(None, 0), (None, None)])
@pytest.mark.parametrize("ascending,nulls_first", [(True, True), (False, False), (True, False)])
def test_aliases_equal_the_range_frames(lower, upper, ascending, nulls_first):
    rng = np.random.default_rng(5)
    n = 300
    p = np.sort(rng.integers(0, 7, n))
    part, order = [], []
    for g in np.unique(p):
        k = int((p == g).sum())
        o = sorted([None if rng.random() < 0.2 else int(x) for x in rng.integers(0, 9, k)],
                   key=lambda x: ((x is None) != nulls_first, 0 if x is None else (x if ascending else -x)))
        part += [(int(g),)] * k
        order += [(x,) for x in o]
    vals = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-10 ** 17, 10 ** 17, n)]
    for kind, vt in ((W.SUM, "decimal"), (W.COUNT, "int"), (W.COUNT_ALL, "int"), (W.MIN, "int"), (W.MAX, "int")):
        exp = W.evaluate(part, order, kind, vals, vtype=vt, frame=W.RANGE, lower=lower, upper=upper, precision=18)
        got = R.evaluate(part, order, kind, vals, vtype=vt, lower=lower, upper=upper, ascending=ascending, nulls_first=nulls_first, precision=18)
        assert got == exp, kind


def test_distinct_timestamps_match_pandas_time_rolling():
    pd = pytest.importorskip("pandas")
    rng = np.random.default_rng(11)
    rows = []
    for g in range(6):
        ts = np.sort(rng.choice(10 ** 6, size=int(rng.integers(1, 80)), replace=False))
        rows += [(g, int(t)) for t in ts]
    p = np.array([r[0] for r in rows])
    ts = np.array([r[1] for r in rows], dtype=np.int64)
    v = rng.integers(-1000, 1000, len(rows)).astype(np.float64)
    part, order, vals = [(int(x),) for x in p], [(int(x),) for x in ts], [float(x) for x in v]
    for k in (0, 1, 1000, 50000, 10 ** 6):
        df = pd.DataFrame({"p": p, "ts": pd.to_datetime(ts, unit="us"), "v": v})
        roll = df.groupby("p").rolling(pd.Timedelta(microseconds=k), on="ts", closed="both")
        exp_sum = roll["v"].sum().to_numpy()
        exp_cnt = roll["v"].count().to_numpy()
        assert R.evaluate(part, order, W.SUM, vals, vtype="float", lower=-k, upper=0) == [float(x) for x in exp_sum], k
        assert R.evaluate(part, order, W.COUNT, vals, lower=-k, upper=0) == [int(x) for x in exp_cnt], k
