"""Row-at-a-time restatement of Spark's window functions over a batch sorted by (partition keys, order keys).

Sequential, as Spark's WindowExec frame classes are (sql/core .../window/WindowFunctionFrame.scala: the unbounded-preceding
frame grows row by row, the sliding frame is re-evaluated per row).  It stands for the GPU path of the reference:
GpuWindowExpression.scala:531 (GpuSpecifiedWindowFrame), :1367-1600 (SumBinaryFixer: a running decimal sum stays NULL for
the rest of the partition once it overflowed, comment near :1520), :1645 / :1772 (RankFixer, DenseRankFixer), :1912-2110 (rank,
dense_rank, row_number, lead, lag).

Values are Python values with None for NULL: ints (decimals unscaled), floats.  Integer SUM wraps like Java's long, decimal
sums are exact Python ints, float sums run left to right from 0.0.  Keys are equal when their normalised forms are: NULL = NULL,
NaN = NaN, -0.0 = 0.0.
"""
import math

ROW_NUMBER, RANK, DENSE_RANK, LEAD, LAG = 1, 2, 3, 4, 5
SUM, COUNT, COUNT_ALL, MIN, MAX = 10, 11, 12, 13, 14
ROWS, RANGE = 0, 1


def _norm(v):
    if isinstance(v, float):
        if math.isnan(v):
            return ("nan",)
        if v == 0.0:
            return 0.0
    return v


def _key(row):
    return tuple(_norm(v) for v in row)


def groups(part_keys, order_keys):
    """-> (partition start of each row, peer-group start of each row, partition end of each row, peer-group end of each row)"""
    n = len(part_keys)
    ps, qs = [0] * n, [0] * n
    for i in range(n):
        if i == 0 or _key(part_keys[i]) != _key(part_keys[i - 1]):
            ps[i] = qs[i] = i
        else:
            ps[i] = ps[i - 1]
            qs[i] = qs[i - 1] if _key(order_keys[i]) == _key(order_keys[i - 1]) else i
    pe, qe = [0] * n, [0] * n
    for i in reversed(range(n)):
        pe[i] = pe[i + 1] if i + 1 < n and ps[i + 1] == ps[i] else i
        qe[i] = qe[i + 1] if i + 1 < n and qs[i + 1] == qs[i] else i
    return ps, qs, pe, qe


def _wrap64(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= 1 << 63 else v


class _Frame:
    """the aggregate state of one frame, grown row by row (the unbounded-preceding frame of Spark's WindowExec extends its
    state; a sliding frame is rebuilt)"""

    def __init__(self, vtype, precision):
        self.vtype, self.lim = vtype, 10 ** precision
        self.rows = self.count = 0
        self.acc = 0.0 if vtype == "float" else 0
        self.overflow = False
        self.lo = self.hi = None
        self.nan = False

    def add(self, v):
        self.rows += 1
        if v is None:
            return
        self.count += 1
        if self.vtype == "float":
            self.acc += v
        elif self.vtype == "decimal":
            self.acc += v
            self.overflow = self.overflow or abs(self.acc) >= self.lim   # SumBinaryFixer: sticky for a running frame
        elif isinstance(v, int):
            self.acc = _wrap64(self.acc + v)
        n = _norm(v)
        if n == ("nan",):
            self.nan = True   # Spark's float order: NaN greatest
        else:
            self.lo = n if self.lo is None else min(self.lo, n)
            self.hi = n if self.hi is None else max(self.hi, n)

    def result(self, kind, running):
        if kind == COUNT_ALL:
            return self.rows
        if kind == COUNT:
            return self.count
        if self.count == 0:
            return None
        if kind == MIN:
            return self.lo if self.lo is not None else math.nan
        if kind == MAX:
            return math.nan if self.nan else self.hi
        if self.vtype == "decimal":
            bad = self.overflow if running else abs(self.acc) >= self.lim
            return None if bad else self.acc
        return self.acc


def evaluate(part_keys, order_keys, kind, values=None, vtype="int", frame=ROWS, lower=None, upper=0, offset=1, default=None,
             precision=38):
    """one window function over the sorted rows.  part_keys / order_keys: one tuple per row.  vtype: "int", "float",
    "decimal" or "other".  lower / upper: ROWS offsets, None = UNBOUNDED.  precision: a decimal SUM's result precision."""
    n = len(part_keys)
    ps, qs, pe, qe = groups(part_keys, order_keys)
    out = [None] * n
    cur = None   # [s, e, state] of the last frame
    for i in range(n):
        if kind == ROW_NUMBER:
            out[i] = i - ps[i] + 1
        elif kind == RANK:
            out[i] = qs[i] - ps[i] + 1
        elif kind == DENSE_RANK:
            out[i] = 1 if qs[i] == ps[i] else (out[i - 1] + (qs[i] == i))
        elif kind in (LEAD, LAG):
            j = i + offset if kind == LEAD else i - offset
            out[i] = values[j] if ps[i] <= j <= pe[i] else default
        else:
            running = lower is None and upper == 0
            s = ps[i] if lower is None else max(ps[i], i + lower)
            if frame == RANGE and upper == 0:
                e = qe[i]
            else:
                e = pe[i] if upper is None else min(pe[i], i + upper)
            if not (cur is not None and cur[0] == s and cur[1] <= e):
                cur = [s, s - 1, _Frame(vtype, precision)]
            while cur[1] < e:
                cur[1] += 1
                cur[2].add(values[cur[1]] if values is not None else 0)
            out[i] = cur[2].result(kind, running)
    return out
