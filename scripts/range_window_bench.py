"""What a RANGE frame with a value offset costs on the 16 SF10 lineitem batches of benchdata.tpch.q3_chunk (60 M rows), resident on
the device, sorted by l_shipdate and cut into 16 batches again:

  sum(l_extendedprice), max(l_extendedprice) OVER (ORDER BY l_shipdate RANGE BETWEEN 6 PRECEDING AND CURRENT ROW)

with no PARTITION BY, so the exec holds the whole input as one group.  About 24 k rows share a ship date, so each frame holds
about 170 k rows: the SUM is a difference of prefixes, the MAX a range query over per-tile prefixes and suffixes and a sparse
table of tile maxima.  Reported: wall ms (host clock around the exec and a device synchronise, profiler off, median of --reps
after a warm-up run), kernel ms from a separate profiled run, the largest b2_device_bytes_in_use seen after any next() with every
output batch released at once (the resident input batches included), and the card and its power limit, read in the same run.
--dump writes a digest of every output column (values of valid rows, and validity), so that two builds can be compared.  One
JSON line.

  python scripts/range_window_bench.py [--sf 10] [--reps 3] [--dump out.json]
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bounded_window_bench import column_digest, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dump", default=None)
    a = ap.parse_args()
    import spark_rapids_b200 as m
    from spark_rapids_b200 import execs as E
    from spark_rapids_b200._lib import lib
    from benchdata import tpch
    m.init(0)
    raw = []
    for i in range(tpch.Q3_CHUNKS["lineitem"]):
        c = tpch.q3_chunk("lineitem", a.sf, i)
        raw.append(m.Table.from_columns([m.Column.from_numpy(c["l_extendedprice"], m.DECIMAL64, scale=2),
                                         m.Column.from_numpy(c["l_shipdate"], m.DATE32)]))
    order = [(1, 1, 1)]
    whole = E.GpuSortExec(order, E.GpuBatchSource(raw)).collect()
    del raw
    rows = whole.num_rows
    cuts = [rows * k // 16 for k in range(17)]
    batches = [m.slice_table(whole, cuts[k], cuts[k + 1]) for k in range(16)]
    del whole
    fr = m.range_between(-6, 0)
    funcs = [m.win_sum(0, fr, m.DECIMAL128, 22), m.win_max(0, fr)]
    info = gpu_info()
    m.sync()
    base = m.device_bytes_in_use()
    walls, peak = [], 0
    for _ in range(a.reps + 1):   # the first run warms up
        ex = E.GpuWindowExec(E.GpuBatchSource(batches), [], order, funcs)
        m.sync()
        t0 = time.perf_counter()
        while True:
            b = ex.next()
            if b is None:
                break
            peak = max(peak, m.device_bytes_in_use())
            del b   # released at once: the peak is what the node holds, not the output so far
        m.sync()
        walls.append((time.perf_counter() - t0) * 1e3)
        del ex
    m.profile_enable(True)
    ex = E.GpuWindowExec(E.GpuBatchSource(batches), [], order, funcs)
    outs = list(ex)
    m.sync()
    rep = m.profile_report()
    m.profile_enable(False)
    kern_ms = sum(k["ms"] for k in rep)
    res = {"rows": rows, "batches_in": len(batches), "batches_out": len(outs), "wall_ms": round(float(np.median(walls[1:])), 2),
           "wall_ms_runs": [round(w, 2) for w in walls[1:]], "kernel_ms": round(kern_ms, 2), "input_bytes": base,
           "peak_bytes_in_use": peak, "kernels": {k["name"]: round(k["ms"], 2) for k in rep}, "gpu": info}
    if a.dump:
        digests = []
        for c in range(outs[0].num_columns):
            hv, hd = hashlib.sha256(), hashlib.sha256()
            for b in outs:
                column_digest(m, lib, b.column(c), hv, hd)
            digests.append([hv.hexdigest(), hd.hexdigest()])
        with open(a.dump, "w") as f:
            json.dump({"rows": rows, "columns": digests}, f)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
