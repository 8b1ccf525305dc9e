"""Row-at-a-time restatement of FIRST / LAST / NTH_VALUE with and without IGNORE NULLS, on top of oracle/spark_window.py.

Spark's First / Last / NthValue window functions over the frame [s, e] of each row (sql/core .../window/WindowFunctionFrame.scala;
the GPU plugin's GpuFirst / GpuLast / GpuNthValue, aggregateFunctions.scala): FIRST is the value at s, LAST the value at e and
NTH_VALUE(n) the value at s + n - 1, NULL when the frame is empty or holds fewer than n rows.  With IGNORE NULLS the rows whose
value is NULL are skipped: the first, last or n-th non-NULL value of the frame, NULL when there is none.

The frames are spark_window's (ROWS, and RANGE running) or given explicitly, e.g. by window_range_oracle.frames for value
offsets.  `source_rows` answers with the row a result is copied from (None: NULL), so that a test can compare the copied bytes.
"""
import bisect

from oracle import spark_window as W

FIRST, LAST, NTH_VALUE = 15, 16, 17


def frames(part_keys, order_keys, frame=W.ROWS, lower=None, upper=0):
    """-> [(s, e)] of every row, as spark_window.evaluate finds them (s > e: empty); lower / upper None = UNBOUNDED"""
    n = len(part_keys)
    ps, _, pe, qe = W.groups(part_keys, order_keys)
    out = []
    for i in range(n):
        s = ps[i] if lower is None else max(ps[i], i + lower)
        if frame == W.RANGE and upper == 0:
            e = qe[i]
        else:
            e = pe[i] if upper is None else min(pe[i], i + upper)
        out.append((s, e))
    return out


def source_rows(frames_, kind, valid, n=1, ignore_nulls=False):
    """the row each result comes from, or None; valid[j]: row j's value is not NULL.  The rows that count, in order, are
    `counted`; those of the frame [s, e] are counted[a:b]"""
    counted = [j for j in range(len(valid)) if valid[j] or not ignore_nulls]
    out = []
    for s, e in frames_:
        a, b = bisect.bisect_left(counted, s), bisect.bisect_right(counted, e)
        if kind == LAST:
            out.append(counted[b - 1] if b > a else None)
        else:
            k = 1 if kind == FIRST else n
            out.append(counted[a + k - 1] if k <= b - a else None)
    return out


def over_frames(frames_, kind, values, n=1, ignore_nulls=False):
    """the function over given frames [(s, e)]; values: Python values with None for NULL"""
    src = source_rows(frames_, kind, [v is not None for v in values], n, ignore_nulls)
    return [None if j is None else values[j] for j in src]


def evaluate(part_keys, order_keys, kind, values, frame=W.ROWS, lower=None, upper=0, n=1, ignore_nulls=False):
    """one value function over the sorted rows (part_keys / order_keys: one tuple per row)"""
    return over_frames(frames(part_keys, order_keys, frame, lower, upper), kind, values, n, ignore_nulls)
