"""Row-at-a-time restatement of RANGE frames with value offsets (B2_FRAME_RANGE_VALUE), on top of oracle/spark_window.py.

Spark's RangeBoundOrdering (sql/core .../window/BoundOrdering.scala) with the bound values computed exactly, as the GPU plugin
does (BasicWindowCalc.scala:169-219): for row i with ORDER BY value v, Lb = v + lower and Ub = v + upper (ASC) or v - lower and
v - upper (DESC), in Python ints, so they never wrap; both are NULL when v is NULL.  Within the partition the frame is [s, e]:
s = the first row whose value sorts at or after Lb, e = the last row whose value sorts at or before Ub, where NULL sorts where
nulls_first puts it and equals NULL.  lower / upper None = the partition's edge; 0 = the edge of the row's peer group (over any
ORDER BY, several columns or STRING included).  s > e: the empty frame.  Aggregates are spark_window's _Frame, so SUM, MIN and
MAX are NULL and COUNT and COUNT(*) 0 on an empty frame; a decimal SUM is sticky-NULL only for (None, 0), the running frame.
"""
from oracle import spark_window as W

RANGE_VALUE = 2


def frames(part_keys, order_keys, lower, upper, ascending=True, nulls_first=True):
    """-> [(s, e)] of every row; order_keys: one tuple per row, the first element is the value the offsets apply to"""
    n = len(part_keys)
    ps, qs, pe, qe = W.groups(part_keys, order_keys)

    def at_or_after(x, b):   # x sorts at or after b
        if x is None:
            return not nulls_first
        return x >= b if ascending else x <= b

    def at_or_before(x, b):
        if x is None:
            return nulls_first
        return x <= b if ascending else x >= b

    out = []
    for i in range(n):
        v = order_keys[i][0] if order_keys[i] else None
        if lower is None:
            s = ps[i]
        elif lower == 0 or v is None:
            s = qs[i]
        else:
            lb = v + lower if ascending else v - lower
            s = next((j for j in range(ps[i], pe[i] + 1) if at_or_after(order_keys[j][0], lb)), pe[i] + 1)
        if upper is None:
            e = pe[i]
        elif upper == 0 or v is None:
            e = qe[i]
        else:
            ub = v + upper if ascending else v - upper
            e = next((j for j in range(pe[i], ps[i] - 1, -1) if at_or_before(order_keys[j][0], ub)), ps[i] - 1)
        out.append((s, e))
    return out


def evaluate(part_keys, order_keys, kind, values=None, vtype="int", lower=None, upper=0, ascending=True, nulls_first=True, precision=38):
    """one aggregate (SUM, COUNT, COUNT_ALL, MIN, MAX) over RANGE BETWEEN lower AND upper, by value"""
    fr = frames(part_keys, order_keys, lower, upper, ascending, nulls_first)
    return aggregate(fr, kind, values, vtype, lower is None and upper == 0, precision)


def aggregate(frames_, kind, values=None, vtype="int", running=False, precision=38):
    """one aggregate over given frames [(s, e)]; running: the sticky decimal rule of the (UNBOUNDED, 0) frame"""
    out = []
    cur = None   # [s, e, state] of the last frame, extended while s stays
    for s, e in frames_:
        if not (cur is not None and cur[0] == s and cur[1] <= e):
            cur = [s, s - 1, W._Frame(vtype, precision)]
        while cur[1] < e:
            cur[1] += 1
            cur[2].add(values[cur[1]] if values is not None else 0)
        out.append(cur[2].result(kind, running))
    return out
