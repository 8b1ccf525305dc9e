"""What FIRST / LAST / NTH_VALUE cost through GpuWindowExec, on device-resident batches of about 1 GB: an INT32 partition key
(partitions of --plen rows, which cross batch edges), an INT64 order key (the row's position) and an INT64 value that is 90 % NULL,
--batches batches of --rows rows (default 10 x 50 M = 500 M rows, 20.1 B per row).

  forward fill: last_value(v) IGNORE NULLS OVER (PARTITION BY k ORDER BY t ROWS UNBOUNDED PRECEDING), a running plan carried across
                batches, against SUM(v) over the same frame, the two alternated in one process
  nth_value(v, 3) IGNORE NULLS OVER (... ROWS BETWEEN k PRECEDING AND CURRENT ROW) for k in 8, 1024, 2^20: bounded plans with
                k + 1 rows of context per batch; a select on the rank directory, so the time should not grow with k

Reported per case: wall ms (host clock around the exec and a device synchronise, profiler off, median of --reps after a warm-up
run) and rows per second; the card, its power limit and its max SM clock, read in the same run.  The first two batches of one run
of each case are checked against a numpy restatement.  One JSON line.

  python scripts/value_window_bench.py [--rows 50000000] [--batches 10] [--plen 100000] [--reps 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bounded_window_bench import gpu_info  # noqa: E402


def make_batches(m, rows, nb, plen, seed):
    """the device batches, and host copies of the first two (key, valid, value) for the check"""
    rng = np.random.default_rng(seed)
    out, host = [], []
    for b in range(nb):
        pos = np.arange(b * rows, (b + 1) * rows, dtype=np.int64)
        key = (pos // plen).astype(np.int32)
        valid = rng.random(rows) < 0.1
        val = rng.integers(-10 ** 9, 10 ** 9, rows)
        out.append(m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(pos), m.Column.from_numpy(val, m.INT64, valid)]))
        if b < 2:
            host.append((key, valid, val))
    return out, host


def expected(host, kind, k=None):
    """(values, valid) over the first two batches: numpy restatements of the forward fill, the running SUM and NTH_VALUE(3)
    IGNORE NULLS over ROWS k PRECEDING .. CURRENT ROW"""
    key = np.concatenate([h[0] for h in host])
    valid = np.concatenate([h[1] for h in host])
    val = np.concatenate([h[2] for h in host])
    n = len(key)
    idx = np.arange(n)
    ps = np.searchsorted(key, key, side="left")             # the partition's first row
    if kind == "sum":
        c = np.cumsum(np.where(valid, val, 0))
        s = c - np.where(ps > 0, c[np.maximum(ps - 1, 0)], 0)
        cnt = np.cumsum(valid)
        nv = cnt - np.where(ps > 0, cnt[np.maximum(ps - 1, 0)], 0)
        return s, nv > 0
    if kind == "ffill":
        last = np.maximum.accumulate(np.where(valid, idx, -1))
        ok = last >= ps
        return val[np.maximum(last, 0)], ok
    s = np.maximum(ps, idx - k)
    cnt = np.cumsum(valid)                                     # counted rows in [0, i]
    before = np.where(s > 0, cnt[np.maximum(s - 1, 0)], 0)
    target = before + 3                                        # the 3rd counted row from s, 1-based rank
    pos = np.nonzero(valid)[0]
    ok = target <= cnt
    src = pos[np.minimum(target, len(pos)) - 1]
    return val[src], ok


def run(m, E, batches, funcs, keep_first=0):
    """one pass of the exec: wall ms, and the first keep_first output columns of the function"""
    ex = E.GpuWindowExec(E.GpuBatchSource(batches), [0], [(1, 1, 1)], funcs)
    kept = []
    m.sync()
    t0 = time.perf_counter()
    while True:
        b = ex.next()
        if b is None:
            break
        if len(kept) < keep_first:
            kept.append(b.column(3).to_numpy())
        del b
    m.sync()
    return (time.perf_counter() - t0) * 1e3, kept


def check(kept, exp):
    vals = np.concatenate([k[0] for k in kept])
    ok = np.concatenate([np.asarray(k[1], dtype=bool) for k in kept])
    ev, eok = exp
    return bool(np.array_equal(ok, eok) and np.array_equal(vals[ok], ev[eok]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--plen", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import spark_rapids_b200 as m
    from spark_rapids_b200 import execs as E
    m.init(0)
    info = gpu_info()
    batches, host = make_batches(m, a.rows, a.batches, a.plen, 11)
    total = a.rows * a.batches
    cases = {"ffill": [m.last_value(2, m.rows(None, 0), True)], "running_sum": [m.win_sum(2, m.rows(None, 0))]}
    ks = [8, 1024, 1 << 20]
    for k in ks:
        cases["nth3_k%d" % k] = [m.nth_value(2, 3, m.rows(-k, 0), True)]
    walls = {c: [] for c in cases}
    checks = {}
    for c, funcs in cases.items():   # warm-up, and the check against numpy
        _, kept = run(m, E, batches, funcs, keep_first=2 if len(host) == 2 else 0)
        if kept:
            exp = expected(host, "sum" if c == "running_sum" else "ffill" if c == "ffill" else "nth", int(c[6:]) if c.startswith("nth") else None)
            checks[c] = check(kept, exp)
        del kept
    for _ in range(a.reps):          # the cases alternated
        for c, funcs in cases.items():
            walls[c].append(run(m, E, batches, funcs)[0])
    res = {"rows": total, "batches": a.batches, "input_bytes": int(m.device_bytes_in_use()), "gpu": info, "checks": checks}
    for c in cases:
        med = float(np.median(walls[c]))
        res[c] = {"wall_ms": round(med, 1), "wall_ms_runs": [round(w, 1) for w in walls[c]], "rows_per_s": round(total / med * 1e3)}
    res["ffill_over_sum"] = round(res["ffill"]["wall_ms"] / res["running_sum"]["wall_ms"], 3)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
