"""What the GPU merge of sorted runs and the out-of-core sort cost, against the paths they stand beside.

  (a) b2_merge_sorted (merge-path tree) against order_by(concat(runs)) (the radix re-sort it replaced), for k = 2 and 8 sorted
      runs of an INT64 key and an INT64 payload, 100 M rows in all.  Wall ms per call (host clock around the call and a
      device synchronise, profiler off, the two paths alternated), per-kernel ms (profiler on, separate call), the HBM bytes
      the merge algorithm needs (computed from the shapes, below) and their rate against the 3.35 TB/s H100 SXM data sheet.
      The two outputs are checked identical.
  (b) the 16 SF10 lineitem batches of benchdata.tpch.q3_chunk, resident on the device, sorted by (l_shipdate, l_orderkey):
      the single-batch GpuSortExec against the out-of-core one at a 1 GiB target, alternated; wall ms, output batches, bytes
      spilled.  The outputs are checked identical.
  (c) the same batches fed from host memory under an allocation limit of half the input.  The window of an out-of-core round
      holds about three copies of the target (pieces, concatenation, merged result), so the target here is 128 MiB; the
      single-batch path is run once to show it cannot finish.

The card, its power limit and its SM clock are read in the same run.  One JSON line per measurement.

  python scripts/out_of_core_sort_bench.py [--rows 100000000] [--reps 3] [--sf 10] [--skip a,b,c]
"""
import argparse
import gc
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0     # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def merge_bytes(n, k):
    """HBM bytes b2_merge_sorted needs for n rows of (INT64 key, INT64 payload) in k runs of equal size:
    concatenation (read + write 16 B/row), first key chunk (read 8, write 8), identity map (write 4), per merge level read
    key + row (12) and write both (12) except the last level, which writes the row only (4), and the gather (map 4, read 16,
    write 16).  Returns (total, merge-kernel share)."""
    levels = max(1, math.ceil(math.log2(k)))
    kern = levels * 12 * n + (levels - 1) * 12 * n + 4 * n
    return 32 * n + 16 * n + 4 * n + kern + 36 * n, kern


def timed(m, f):
    m.sync()
    t0 = time.perf_counter()
    out = f()
    m.sync()
    return (time.perf_counter() - t0) * 1e3, out


def kernel_ms(m, f):
    m.profile_enable(True)
    try:
        out = f()
        m.sync()
        rep = {k["name"]: round(k["ms"], 3) for k in m.profile_report()}
    finally:
        m.profile_enable(False)
    del out
    return rep


def bench_merge(m, rows, reps, info):
    key = [(0, 1, 1)]
    for k in (2, 8):
        rng = np.random.default_rng(k)
        per = rows // k
        runs = []
        for r in range(k):
            kv = np.sort(rng.integers(-2**62, 2**62, per, dtype=np.int64))
            runs.append(m.Table.from_columns([m.Column.from_numpy(kv), m.Column.from_numpy(np.arange(r * per, (r + 1) * per, dtype=np.int64))]))
        n = per * k
        paths = {"merge": lambda: m.merge_sorted(runs, key), "resort": lambda: m.order_by(m.concat(runs), key)}
        ms = {p: [] for p in paths}
        same = None
        for rep in range(reps + 1):        # rep 0 warms both paths up and checks them
            order = list(paths) if rep % 2 == 0 else list(paths)[::-1]
            outs = {}
            for p in order:
                t, out = timed(m, paths[p])
                if rep:
                    ms[p].append(round(t, 2))
                if rep == 0:
                    outs[p] = [out.column(c).to_numpy()[0] for c in range(2)]
                del out
            if rep == 0:
                same = all(np.array_equal(a, b) for a, b in zip(outs["merge"], outs["resort"]))
                del outs
            gc.collect()
        kms = {p: kernel_ms(m, paths[p]) for p in paths}
        total, kern = merge_bytes(n, k)
        mk = sum(v for name, v in kms["merge"].items() if name.startswith("merge_path"))
        med = float(np.median(ms["merge"]))
        print(json.dumps({"case": "a", "runs": k, "rows": n, "identical": same, "wall_ms": ms, "kernel_ms": kms,
                          "merge_algorithmic_bytes": total, "merge_kernel_bytes": kern,
                          "merge_wall_share_of_hbm": round(total / (med * 1e-3) / (HBM_GBS * 1e9), 3),
                          "merge_kernel_share_of_hbm": round(kern / (mk * 1e-3) / (HBM_GBS * 1e9), 3) if mk else None, "gpu": info}), flush=True)
        del runs, paths
        gc.collect()


def bench_lineitem(m, sf, reps, info, skip):
    import bench
    from benchdata import tpch
    from spark_rapids_b200 import execs as E
    cols = bench.Q3_SCHEMA["lineitem"]
    types = [bench.q3_dtype(m, c) for c in cols]
    chunks = [tpch.q3_chunk("lineitem", sf, i) for i in range(tpch.Q3_CHUNKS["lineitem"])]
    keys = [(cols.index("l_shipdate"), 1, 1), (cols.index("l_orderkey"), 1, 1)]
    in_bytes = sum(ch[c].nbytes for ch in chunks for c in cols)
    ref = None
    if "b" not in skip:
        dev = [m.Table.from_columns([m.Column.from_numpy(ch[c], dtype=dt, scale=s) for c, (dt, s) in zip(cols, types)]) for ch in chunks]

        def single():
            out = E.GpuSortExec(keys, E.GpuBatchSource(dev)).collect()
            return [out]

        def ooc():
            node = E.GpuSortExec(keys, E.GpuBatchSource(dev), target_bytes=1 << 30)
            return list(node)

        ms = {"single": [], "out_of_core": []}
        nb, spilled = None, None
        for rep in range(reps + 1):
            order = ["single", "out_of_core"] if rep % 2 == 0 else ["out_of_core", "single"]
            outs = {}
            for p in order:
                s0 = m.memory_stats()["spilled_bytes"]
                t, out = timed(m, single if p == "single" else ooc)
                if p == "out_of_core":
                    nb, spilled = len(out), m.memory_stats()["spilled_bytes"] - s0
                if rep:
                    ms[p].append(round(t, 1))
                else:
                    outs[p] = [np.concatenate([b.column(c).to_numpy()[0] for b in out]) for c in range(len(cols))]
                del out
                gc.collect()
            if rep == 0:
                same = all(np.array_equal(a, b) for a, b in zip(outs["single"], outs["out_of_core"]))
                ref = outs["single"]
                del outs
        print(json.dumps({"case": "b", "sf": sf, "rows": sum(len(ch[cols[0]]) for ch in chunks), "input_bytes": in_bytes, "identical": same,
                          "wall_ms": ms, "out_of_core_batches": nb, "out_of_core_spilled_bytes": spilled, "gpu": info}), flush=True)
        del dev
        gc.collect()
    if "c" not in skip:
        def host():
            return E.GpuHostBatchSource([[(dt, s, ch[c], None) for c, (dt, s) in zip(cols, types)] for ch in chunks])

        m.sync()
        limit = m.device_bytes_in_use() + in_bytes // 2
        m.set_alloc_limit(limit)
        try:
            try:
                E.GpuSortExec(keys, host()).collect()
                single = "finished"
            except m.B2Error as e:
                single = "error %d" % e.code
            gc.collect()
            s0 = m.memory_stats()["spilled_bytes"]
            got = [[] for _ in cols]

            def run():
                nbat = 0
                for b in E.GpuSortExec(keys, host(), target_bytes=128 << 20):
                    for c in range(len(cols)):
                        got[c].append(b.column(c).to_numpy()[0])
                    nbat += 1
                return nbat
            t, nbat = timed(m, run)
            spilled = m.memory_stats()["spilled_bytes"] - s0
        finally:
            m.set_alloc_limit(0)
        same = None if ref is None else all(np.array_equal(np.concatenate(g), r) for g, r in zip(got, ref))
        print(json.dumps({"case": "c", "sf": sf, "input_bytes": in_bytes, "alloc_limit_headroom": in_bytes // 2, "single_batch": single,
                          "out_of_core_target": 128 << 20, "out_of_core_wall_ms_incl_d2h_of_output": round(t, 1), "out_of_core_batches": nbat,
                          "spilled_bytes": spilled, "identical_to_b": same, "gpu": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--skip", default="")
    a = ap.parse_args()
    skip = set(a.skip.split(",")) if a.skip else set()
    import spark_rapids_b200 as m
    m.init(0)
    info = gpu_info()
    if "a" not in skip:
        bench_merge(m, a.rows, a.reps, info)
    if not {"b", "c"} <= skip:
        bench_lineitem(m, a.sf, a.reps, info, skip)


if __name__ == "__main__":
    main()
