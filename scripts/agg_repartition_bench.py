"""What repartitioning the hash aggregate's merge costs, against the single merge it stands beside.

Workloads (inputs generated here, resident on the device):
  q3       the shape of the SF100 q3 group-by: 31.3 M rows in 4 batches of [l_orderkey INT64, o_orderdate DATE32, o_shippriority
           INT32, price DECIMAL64(12,2), discount DECIMAL64(12,2)] over 12.9 M (orderkey, date, priority) groups, COMPLETE mode,
           SUM(price * (1 - discount)) as DECIMAL128(36,4): the aggregate of bench.py's q3 plan
  highcard 200 M rows in 8 batches of [INT64 key, INT64 value] over 10^8 keys, COMPLETE mode, SUM(value) and COUNT(*)
Arms: the default single merge, and targets of 4 GiB, 1 GiB and 256 MiB (16 buckets).  Per arm: wall ms (host clock around the
whole pull and a device synchronise, profiler off; the arms alternated over the repetitions), kernel ms per kernel (profiler
on, a separate call), the repartition stats, the bytes the split kernels need and their rate against the 3.35 TB/s H100 SXM
data sheet, and whether the output sorted by key is identical to the default arm's.  One more arm feeds highcard from host
memory under an allocation limit of 3 GiB above the base: the single merge fails there, the 256 MiB target finishes.

The card, its power limit and its SM clock are read in the same run.  One JSON line per measurement.

  python scripts/agg_repartition_bench.py [--reps 3] [--skip q3,highcard,limit]
"""
import argparse
import ctypes
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0     # H100 SXM data sheet
TARGETS = {"default": None, "4GiB": 4 << 30, "1GiB": 1 << 30, "256MiB": 256 << 20}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def raw(m, c):
    """a column's values as int64 words per row (DECIMAL128: two), NULLs as 0 and a flag"""
    ci = c.info()
    n = ci.size
    w = 2 if ci.dtype == m.DECIMAL128 else 1
    width = {m.INT32: 4, m.DATE32: 4}.get(ci.dtype, 8)
    data = np.zeros(n * width * w, dtype=np.uint8)
    vb = np.zeros((n + 7) // 8, dtype=np.uint8)
    m.check(m.lib.b2_column_to_host(c.h, data.ctypes.data_as(ctypes.c_void_p), vb.ctypes.data_as(ctypes.c_void_p), None))
    vals = data.view(np.int32).astype(np.int64) if width == 4 else data.view(np.int64)
    return vals.reshape(n, w), m.unpack_bits(vb, n)


def sorted_output(m, batches, nkeys):
    """all output rows as one int64 matrix (NULL values zeroed, a validity word per column), sorted by the key columns"""
    parts = []
    for t in batches:
        cols = []
        for i in range(t.num_columns):
            v, ok = raw(m, t.column(i))
            cols += [np.where(ok[:, None], v, 0), ok[:, None].astype(np.int64)]
        parts.append(np.concatenate(cols, axis=1))
    a = np.concatenate(parts) if parts else np.zeros((0, 1), np.int64)
    return a[np.lexsort([a[:, k] for k in range(2 * nkeys - 1, -1, -1)])]


def q3_workload(m):
    rng = np.random.default_rng(3)
    rows, groups, nb = 31_300_000, 12_900_000, 4
    okey = rng.permutation(np.arange(1, 4 * groups, 4, dtype=np.int64)[:groups])
    which = np.r_[np.arange(groups), rng.integers(0, groups, rows - groups)]
    rng.shuffle(which)
    key = okey[which]
    date = (8800 + key % 1500).astype(np.int32)
    prio = np.zeros(rows, np.int32)
    price = rng.integers(90_000, 10_500_000, rows).astype(np.int64)
    disc = rng.integers(0, 11, rows).astype(np.int64)
    bounds = np.linspace(0, rows, nb + 1).astype(int)
    batches = [m.Table.from_columns([m.Column.from_numpy(key[s:e]), m.Column.from_numpy(date[s:e], dtype=m.DATE32), m.Column.from_numpy(prio[s:e]),
                                     m.Column.from_numpy(price[s:e], dtype=m.DECIMAL64, scale=2), m.Column.from_numpy(disc[s:e], dtype=m.DECIMAL64, scale=2)])
               for s, e in zip(bounds[:-1], bounds[1:])]
    one = m.lit(1, m.DECIMAL32, 1, 0)
    p, d = m.col(3, m.DECIMAL64, 12, 2, nullable=False), m.col(4, m.DECIMAL64, 12, 2, nullable=False)
    prog = m.Program([m.col(0, m.INT64, nullable=False), m.col(1, m.DATE32, nullable=False), m.col(2, m.INT32, nullable=False), p * (one - d)])
    # partial row: 8 + 4 + 4 key bytes, 16 B sum, 8 B count of the decimal SUM
    return dict(batches=batches, prog=prog, keys=[0, 1, 2], specs=[(m.AGG_SUM, 3, m.DECIMAL128, 4, 36)], key_bytes=16, row_bytes=40,
                rows=rows, groups=groups)


def highcard_arrays(rows=200_000_000, groups=100_000_000, nb=8):
    rng = np.random.default_rng(4)
    g = np.r_[np.arange(groups), rng.integers(0, groups, rows - groups)]
    rng.shuffle(g)
    with np.errstate(over="ignore"):
        key = (g.astype(np.int64) * np.int64(-7046029254386353131)) ^ np.int64(0x5DEECE66D)
    val = rng.integers(-10**9, 10**9, rows)
    bounds = np.linspace(0, rows, nb + 1).astype(int)
    return [(key[s:e], val[s:e]) for s, e in zip(bounds[:-1], bounds[1:])], rows, groups


def highcard_workload(m, arrays):
    parts, rows, groups = arrays
    batches = [m.Table.from_columns([m.Column.from_numpy(k), m.Column.from_numpy(v)]) for k, v in parts]
    prog = m.Program([m.col(0, m.INT64, nullable=False), m.col(1, m.INT64, nullable=False)])
    return dict(batches=batches, prog=prog, keys=[0], specs=[(m.AGG_SUM, 1, m.INT64, 0, 0), (m.AGG_COUNT_ALL, 0)], key_bytes=8, row_bytes=24,
                rows=rows, groups=groups)


def node(E, w, src, target):
    kw = {} if target is None else dict(target_bytes=target)
    return E.GpuHashAggregateExec(src, w["keys"], w["specs"], pre_project=w["prog"], mode="complete", **kw)


def split_bytes(stats, key_bytes, row_bytes):
    """bytes the split kernels need for stats['bytes_split'] bytes of pieces: the count pass reads the keys and writes a 1-byte
    bucket id per row; the scatter pass reads the id and the row and writes the row"""
    b = stats["bytes_split"]
    rows = b // row_bytes
    return b * key_bytes // row_bytes + rows + rows + 2 * b


def bench(m, E, name, w, reps, info):
    outs_ref = None
    ms = {a: [] for a in TARGETS}
    for rep in range(reps + 1):
        arms = list(TARGETS) if rep % 2 == 0 else list(TARGETS)[::-1]
        for a in arms:
            n = node(E, w, E.GpuBatchSource(w["batches"]), TARGETS[a])
            m.sync()
            t0 = time.perf_counter()
            out = list(n)
            m.sync()
            dt = (time.perf_counter() - t0) * 1e3
            if rep:
                ms[a].append(round(dt, 1))
            else:
                rec = {"case": name, "arm": a, "target": TARGETS[a], "batches": len(out), "rows": sum(t.num_rows for t in out), "stats": n.repartition_stats}
                s = sorted_output(m, out, len(w["keys"]))
                if a == "default":
                    outs_ref = s
                    rec["identical_to_default"] = True
                else:
                    rec["identical_to_default"] = bool(outs_ref is not None and s.shape == outs_ref.shape and np.array_equal(s, outs_ref))
                del s
                ms.setdefault("first", {})[a] = rec
            del out, n
            gc.collect()
    for a in TARGETS:
        n = node(E, w, E.GpuBatchSource(w["batches"]), TARGETS[a])
        m.profile_enable(True)
        try:
            out = list(n)
            m.sync()
            rep = {}
            for k in m.profile_report():
                rep[k["name"]] = round(rep.get(k["name"], 0) + k["ms"], 3)
        finally:
            m.profile_enable(False)
        del out, n
        gc.collect()
        rec = ms["first"][a]
        sk = round(rep.get("hash_split_count_kernel", 0) + rep.get("hash_split_scatter_kernel", 0), 3)
        need = split_bytes(rec["stats"], w["key_bytes"], w["row_bytes"])
        rec.update({"rows_in": w["rows"], "groups": w["groups"], "wall_ms": ms[a], "kernel_ms_total": round(sum(rep.values()), 2), "kernel_ms": rep,
                    "split_kernel_ms": sk, "split_bytes_needed": need,
                    "split_share_of_hbm": round(need / (sk * 1e-3) / (HBM_GBS * 1e9), 3) if sk else None, "gpu": info})
        print(json.dumps(rec), flush=True)
    return outs_ref


def bench_limit(m, E, arrays, ref, info):
    parts, rows, groups = arrays
    host = [[(m.INT64, 0, k, None), (m.INT64, 0, v, None)] for k, v in parts]
    prog = m.Program([m.col(0, m.INT64, nullable=False), m.col(1, m.INT64, nullable=False)])
    specs = [(m.AGG_SUM, 1, m.INT64, 0, 0), (m.AGG_COUNT_ALL, 0)]
    mk = lambda **kw: E.GpuHashAggregateExec(E.GpuHostBatchSource(host), [0], specs, pre_project=prog, mode="complete", **kw)
    gc.collect()
    m.sync()
    headroom = 3 << 30
    m.set_alloc_limit(m.device_bytes_in_use() + headroom)
    try:
        try:
            mk().collect()
            single = "finished"
        except m.B2Error as e:
            single = "error %d" % e.code
        gc.collect()
        s0 = m.memory_stats()["spilled_bytes"]
        n = mk(target_bytes=256 << 20)
        m.sync()
        t0 = time.perf_counter()
        parts_out = []
        for t in n:
            parts_out.append(sorted_output(m, [t], 1))
            del t
        m.sync()
        dt = (time.perf_counter() - t0) * 1e3
        spilled = m.memory_stats()["spilled_bytes"] - s0
        stats = n.repartition_stats
    finally:
        m.set_alloc_limit(0)
    a = np.concatenate(parts_out)
    a = a[np.lexsort([a[:, 1], a[:, 0]])]
    same = None if ref is None else bool(a.shape == ref.shape and np.array_equal(a, ref))
    print(json.dumps({"case": "highcard_alloc_limit", "alloc_limit_headroom": headroom, "single_merge": single, "target": 256 << 20,
                      "wall_ms_incl_d2h_of_output": round(dt, 1), "spilled_bytes": spilled, "stats": stats, "identical_to_default": same,
                      "gpu": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip", default="")
    a = ap.parse_args()
    skip = set(a.skip.split(",")) if a.skip else set()
    import spark_rapids_b200 as m
    from spark_rapids_b200 import execs as E
    m.init(0)
    info = gpu_info()
    if "q3" not in skip:
        w = q3_workload(m)
        bench(m, E, "q3", w, a.reps, info)
        del w
        gc.collect()
    if not {"highcard", "limit"} <= skip:
        arrays = highcard_arrays()
        ref = None
        if "highcard" not in skip:
            w = highcard_workload(m, arrays)
            ref = bench(m, E, "highcard", w, a.reps, info)
            del w
            gc.collect()
        if "limit" not in skip:
            bench_limit(m, E, arrays, ref, info)


if __name__ == "__main__":
    main()
