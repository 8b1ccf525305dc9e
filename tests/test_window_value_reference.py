"""The FIRST / LAST / NTH_VALUE restatement (tests/window_value_oracle.py) against hand-worked Spark answers, and against a scan of
every frame row by row."""
import numpy as np

from oracle import spark_window as W
from tests import window_range_oracle as R
from tests import window_value_oracle as V


def _keys(xs):
    return [(x,) for x in xs]


# two partitions; the first has a peer group of two rows (order key 2)
P, O = _keys([1, 1, 1, 1, 2, 2]), _keys([1, 2, 2, 3, 1, 1])
VALS = [None, 10, 20, None, 5, None]


def test_default_frame_with_order_by_is_range_running():
    ev = lambda kind, **kw: V.evaluate(P, O, kind, VALS, frame=W.RANGE, lower=None, upper=0, **kw)
    assert ev(V.FIRST) == [None, None, None, None, 5, 5]
    assert ev(V.FIRST, ignore_nulls=True) == [None, 10, 10, 10, 5, 5]
    assert ev(V.LAST) == [None, 20, 20, None, None, None]          # the peer group's last row
    assert ev(V.LAST, ignore_nulls=True) == [None, 20, 20, 20, 5, 5]
    assert ev(V.NTH_VALUE, n=2) == [None, 10, 10, 10, None, None]
    assert ev(V.NTH_VALUE, n=2, ignore_nulls=True) == [None, 20, 20, 20, None, None]


def test_default_frame_without_order_by_is_the_partition():
    ev = lambda kind, **kw: V.evaluate(P, _keys([0] * 6), kind, VALS, lower=None, upper=None, **kw)
    assert ev(V.FIRST) == [None] * 4 + [5, 5]
    assert ev(V.FIRST, ignore_nulls=True) == [10] * 4 + [5, 5]
    assert ev(V.LAST) == [None] * 6
    assert ev(V.LAST, ignore_nulls=True) == [20] * 4 + [5, 5]
    assert ev(V.NTH_VALUE, n=3) == [20] * 4 + [None, None]


def test_ignore_nulls_over_all_null_frames():
    p, o, v = _keys([0] * 5), _keys(range(5)), [None, None, 3, None, None]
    assert V.evaluate(p, o, V.FIRST, v, lower=-1, upper=0, ignore_nulls=True) == [None, None, 3, 3, None]
    assert V.evaluate(p, o, V.LAST, v, lower=-1, upper=0, ignore_nulls=True) == [None, None, 3, 3, None]
    assert V.evaluate(p, o, V.LAST, [None] * 5, lower=None, upper=None, ignore_nulls=True) == [None] * 5


def test_forward_fill():
    p, o = _keys([0] * 4 + [1] * 3), _keys(range(7))
    v = [None, 1, None, None, None, 7, None]
    assert V.evaluate(p, o, V.LAST, v, lower=None, upper=0, ignore_nulls=True) == [None, 1, 1, 1, None, 7, 7]


def test_nth_value_past_the_frame():
    p, o, v = _keys([0] * 4), _keys(range(4)), [1, 2, 3, 4]
    assert V.evaluate(p, o, V.NTH_VALUE, v, lower=-1, upper=1, n=3) == [None, 3, 4, None]
    assert V.evaluate(p, o, V.NTH_VALUE, v, lower=-1, upper=1, n=5) == [None] * 4
    assert V.evaluate(p, o, V.NTH_VALUE, v, lower=None, upper=0, n=2) == [None, 2, 2, 2]


def test_empty_frames_at_a_partition_end():
    p, o, v = _keys([1, 1, 1, 2]), _keys(range(4)), [1, 2, 3, 4]
    assert V.evaluate(p, o, V.FIRST, v, lower=1, upper=4) == [2, 3, None, None]
    assert V.evaluate(p, o, V.LAST, v, lower=1, upper=4) == [3, 3, None, None]
    assert V.evaluate(p, o, V.LAST, v, lower=-5, upper=-1) == [None, 1, 2, None]


def test_range_value_frames_hold_the_trailing_nulls_of_nulls_last():
    p, o, v = _keys([0] * 5), _keys([1, 2, 4, None, None]), [10, None, 30, 40, None]
    to_end = R.frames(p, o, 0, None, True, False)
    assert to_end == [(0, 4), (1, 4), (2, 4), (3, 4), (3, 4)]
    assert V.over_frames(to_end, V.LAST, v) == [None] * 5
    assert V.over_frames(to_end, V.LAST, v, ignore_nulls=True) == [40] * 5
    assert V.over_frames(to_end, V.FIRST, v, ignore_nulls=True) == [10, 30, 30, 40, 40]
    near = R.frames(p, o, -1, 1, True, False)
    assert near == [(0, 1), (0, 1), (2, 2), (3, 4), (3, 4)]
    assert V.over_frames(near, V.FIRST, v) == [10, 10, 30, 40, 40]
    assert V.over_frames(near, V.LAST, v) == [None, None, 30, None, None]
    assert V.over_frames(near, V.LAST, v, ignore_nulls=True) == [10, 10, 30, 40, 40]


def test_source_rows_equal_a_scan_of_each_frame():
    rng = np.random.default_rng(3)
    n = 300
    p = _keys(np.sort(rng.integers(0, 9, n)).tolist())
    o = _keys(rng.integers(0, 4, n).tolist())
    valid = (rng.random(n) < 0.4).tolist()
    for lower, upper in [(None, 0), (-3, 2), (1, 4), (None, None), (-7, -2), (None, 3)]:
        fr = V.frames(p, o, W.ROWS, lower, upper)
        for kind, k in [(V.FIRST, 1), (V.LAST, 1), (V.NTH_VALUE, 2), (V.NTH_VALUE, 5)]:
            for ign in (False, True):
                exp = []
                for s, e in fr:
                    rows = [j for j in range(s, e + 1) if valid[j] or not ign]
                    pick = (rows[-1] if rows else None) if kind == V.LAST else (rows[k - 1] if k <= len(rows) else None)
                    exp.append(pick)
                assert V.source_rows(fr, kind, valid, k, ign) == exp, (lower, upper, kind, k, ign)
