"""What GpuWindowExec costs on the 16 SF10 lineitem batches of benchdata.tpch.q3_chunk (60 M rows), resident on the device and
sorted first by GpuSortExec (timed apart from the window; the full sort hands the window one batch).  Workloads:

  rank       rank() OVER (PARTITION BY l_orderkey ORDER BY l_extendedprice DESC): many small partitions (mode 3 is not needed:
             ranking runs batch by batch with the device carry)
  running    sum(l_extendedprice) OVER (PARTITION BY l_shipdate ORDER BY l_orderkey ROWS UNBOUNDED PRECEDING) and the same with
             Spark's default RANGE frame: about 2.5 K long partitions
  lag_mov7   lag(l_extendedprice, 1) and a 7-row moving sum, no PARTITION BY (the whole input is one group)

For each: wall ms (host clock around the exec and a device synchronise, profiler off), kernel ms from a separate profiled
run, and the algorithmic bytes (key and value columns read once, outputs written once) over kernel time against the 3.35 TB/s
H100 SXM data sheet.  The card and its power limit are read in the same run.  One JSON line per workload.

  python scripts/window_bench.py [--sf 10] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0     # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import spark_rapids_b200 as m
    from spark_rapids_b200 import execs as E
    from benchdata import tpch
    m.init(0)
    batches = []
    for i in range(tpch.Q3_CHUNKS["lineitem"]):
        c = tpch.q3_chunk("lineitem", a.sf, i)
        batches.append(m.Table.from_columns([m.Column.from_numpy(c["l_orderkey"]), m.Column.from_numpy(c["l_extendedprice"], m.DECIMAL64, scale=2),
                                             m.Column.from_numpy(c["l_shipdate"], m.DATE32)]))
    rows = sum(b.num_rows for b in batches)
    info = gpu_info()
    work = {
        "rank": ([0], [(1, 0, 0)], [m.rank()], 8 + 8, 4),
        "running": ([2], [(0, 1, 1)], [m.win_sum(1, m.rows(None, 0), m.DECIMAL128, 22), m.win_sum(1, m.range_running(), m.DECIMAL128, 22)], 4 + 8 + 8, 32),
        "lag_mov7": ([], [(2, 1, 1), (0, 1, 1)], [m.lag(1, 1), m.win_sum(1, m.rows(-6, 0), m.DECIMAL128, 22)], 4 + 8 + 8, 8 + 16),
    }
    for name, (part, order, funcs, in_bytes, out_bytes) in work.items():
        keys = [(c, 1, 1) for c in part] + order
        sorted_batches = list(E.GpuSortExec(keys, E.GpuBatchSource(batches)))   # GpuSortExec below the window, timed apart
        m.sync()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            list(E.GpuSortExec(keys, E.GpuBatchSource(batches)))
            m.sync()
        sort_ms = (time.perf_counter() - t0) * 1e3 / a.reps
        walls = []
        for _ in range(a.reps + 1):   # the first run warms up
            ex = E.GpuWindowExec(E.GpuBatchSource(sorted_batches), part, order, funcs)
            m.sync()
            t0 = time.perf_counter()
            outs = list(ex)
            m.sync()
            walls.append((time.perf_counter() - t0) * 1e3)
            del outs
        m.profile_enable(True)
        ex = E.GpuWindowExec(E.GpuBatchSource(sorted_batches), part, order, funcs)
        outs = list(ex)
        m.sync()
        rep = m.profile_report()
        m.profile_enable(False)
        kern_ms = sum(k["ms"] for k in rep if k["name"].startswith("window_") or k["name"] == "gather_fixed_kernel")
        nbytes = rows * (in_bytes + out_bytes)
        print(json.dumps({"workload": name, "rows": rows, "batches_in": len(sorted_batches), "batches_out": len(outs), "sort_ms": round(sort_ms, 2),
                          "wall_ms": round(float(np.median(walls[1:])), 2), "kernel_ms": round(kern_ms, 2), "algo_bytes": nbytes,
                          "algo_GBps": round(nbytes / kern_ms / 1e6, 1) if kern_ms else None,
                          "hbm_share": round(nbytes / kern_ms / 1e6 / HBM_GBS, 3) if kern_ms else None,
                          "kernels": {k["name"]: round(k["ms"], 2) for k in rep}, "gpu": info}), flush=True)
        del outs, sorted_batches


if __name__ == "__main__":
    main()
