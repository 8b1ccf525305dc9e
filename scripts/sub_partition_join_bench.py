"""What the one-pass hash split and the sub-partitioned hash join cost, against the paths they stand beside.

  (a) b2_hash_split against b2_hash_partition + K b2_slice (murmur_kernel -> partition_table -> K x slice_table) on a q3-shaped
      lineitem batch: 37.5 M rows of an INT64 key and three payload columns (INT64, INT64, nullable INT32), K = 16 and 256.
      Wall ms per call (host clock around the call and a device synchronise, profiler off, the two paths alternated), per-kernel
      ms (profiler on, separate call), the bytes the split algorithm needs (below) and their rate against the 3.35 TB/s H100 SXM
      data sheet.  Every part of the two paths is checked identical.
        count pass:   key bytes in + 1 B bucket id out per row
        scatter pass: 1 B + row bytes in, row bytes out, plus validity in and out (1 bit each) per row
  (b) the SF10 lineitem x orders join on o_orderkey (benchdata.tpch.q3_chunk batches, resident on the device): the single-batch
      GpuShuffledHashJoinExec against the sub-partitioned one at a 256 MiB target, alternated; wall ms, buckets, bytes split.
      The outputs are checked identical as multisets of rows (sorted 64-bit row fingerprints).
  (c) the same join with both sides fed from host memory under an allocation limit of 512 MiB above the base, where only the
      sub-partitioned join finishes, at a 64 MiB target (a pair's hash table takes up to 2x its build bytes rounded up to a power
      of two: at 256 MiB a pair alone needs 512 MiB for it); wall ms (output copied to the host batch by batch) and bytes spilled.

The card, its power limit and its SM clock are read in the same run.  One JSON line per measurement.

  python scripts/sub_partition_join_bench.py [--rows 37500000] [--reps 3] [--sf 10] [--skip a,b,c]
"""
import argparse
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


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


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


def split_bytes(n, key_bytes, row_bytes, nullable_cols):
    count = n * (key_bytes + 1)
    scatter = n * (1 + 2 * row_bytes) + 2 * nullable_cols * n // 8
    return count, scatter


def _same_part(a, b):
    """two parts as [(values, valid)] per column (or None): the same validity, the same values where valid"""
    if a is None or b is None:
        return a is None and b is None
    return all(np.array_equal(ka, kb) and np.array_equal(va[ka], vb[kb]) for (va, ka), (vb, kb) in zip(a, b))


def bench_split(m, rows, reps, info):
    rng = np.random.default_rng(1)
    key = rng.integers(1, 60_000_000, rows).astype(np.int64)
    p1, p2 = rng.integers(0, 10**7, rows).astype(np.int64), rng.integers(0, 11, rows).astype(np.int64)
    p3 = rng.integers(8000, 11000, rows).astype(np.int32)
    t = m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(p1), m.Column.from_numpy(p2),
                              m.Column.from_numpy(p3, valid=rng.random(rows) > 0.01)])
    for k in (16, 256):
        def split():
            return m.hash_split(t, [0], 100, k)

        def partition_slice():
            part, offs = m.hash_partition(t, [0], k, seed=100)
            return [m.slice_table(part, offs[p], offs[p + 1]) if offs[p + 1] > offs[p] else None for p in range(k)]
        paths = {"hash_split": split, "partition_slice": partition_slice}
        ms = {p: [] for p in paths}
        same = None
        for rep in range(reps + 1):
            order = list(paths) if rep % 2 == 0 else list(paths)[::-1]
            outs = {}
            for p in order:
                dt, out = timed(m, paths[p])
                if rep:
                    ms[p].append(round(dt, 2))
                elif k == 16:
                    outs[p] = [None if o is None else [o.column(c).to_numpy() for c in range(4)] for o in out]
                del out
                gc.collect()
            if outs:
                same = all(_same_part(a, b) for a, b in zip(outs["hash_split"], outs["partition_slice"]))
                del outs
        kms = {p: kernel_ms(m, paths[p]) for p in paths}
        cnt_b, sc_b = split_bytes(rows, 8, 28, 1)
        kc, ks = kms["hash_split"].get("hash_split_count_kernel"), kms["hash_split"].get("hash_split_scatter_kernel")
        print(json.dumps({"case": "a", "rows": rows, "parts": k, "identical": same, "wall_ms": ms, "kernel_ms": kms,
                          "count_bytes": cnt_b, "scatter_bytes": sc_b,
                          "count_share_of_hbm": round(cnt_b / (kc * 1e-3) / (HBM_GBS * 1e9), 3) if kc else None,
                          "scatter_share_of_hbm": round(sc_b / (ks * 1e-3) / (HBM_GBS * 1e9), 3) if ks else None, "gpu": info}), flush=True)


def _rows(out_batches, ncols):
    """the output as a multiset of rows: one 64-bit fingerprint per row (odd multipliers per column, wrapping), sorted"""
    fp = np.concatenate([sum(np.asarray(b[c]).astype(np.int64).view(np.uint64) * np.uint64(2 * c + 0x9E3779B97F4A7C15 % 2**63 | 1)
                             for c in range(ncols)) for b in out_batches]) if out_batches else np.zeros(0, np.uint64)
    return [np.sort(fp)]


def bench_join(m, sf, reps, info, skip):
    import bench
    from benchdata import tpch
    from spark_rapids_b200 import execs as E
    side = {}
    for name in ("lineitem", "orders"):
        cols = bench.Q3_SCHEMA[name]
        types = [bench.q3_dtype(m, c) for c in cols]
        side[name] = (cols, types, [tpch.q3_chunk(name, sf, i) for i in range(tpch.Q3_CHUNKS[name])])
    lcols, ocols = side["lineitem"][0], side["orders"][0]
    lk, ok = lcols.index("l_orderkey"), ocols.index("o_orderkey")
    nout = len(lcols) + len(ocols)

    def collect(node):
        outs = [[b.column(c).to_numpy()[0] for c in range(nout)] for b in node]
        return outs

    ref = None
    if "b" not in skip:
        dev = {n: [m.Table.from_columns([m.Column.from_numpy(ch[c], dtype=dt, scale=s) for c, (dt, s) in zip(cols, types)]) for ch in chunks]
               for n, (cols, types, chunks) in side.items()}

        def node(target):
            kw = {} if target is None else dict(target_bytes=target)
            return E.GpuShuffledHashJoinExec([lk], [ok], 0, E.GpuBatchSource(dev["lineitem"]), E.GpuBatchSource(dev["orders"]), **kw)
        ms = {"single": [], "sub_partitioned": []}
        stats, same = None, None
        for rep in range(reps + 1):
            order = ["single", "sub_partitioned"] if rep % 2 == 0 else ["sub_partitioned", "single"]
            outs = {}
            for p in order:
                j = node(None if p == "single" else 256 << 20)
                if rep:
                    dt, out = timed(m, lambda: list(j))
                    ms[p].append(round(dt, 1))
                    del out
                else:
                    outs[p] = _rows(collect(j), nout)
                if p == "sub_partitioned":
                    stats = j.sub_partition_stats
                del j
                gc.collect()
            if rep == 0:
                same = all(np.array_equal(a, b) for a, b in zip(outs["single"], outs["sub_partitioned"]))
                ref = outs["single"]
                del outs
        print(json.dumps({"case": "b", "sf": sf, "identical": same, "wall_ms": ms, "stats": stats, "gpu": info}), flush=True)
        del dev
        gc.collect()
    if "c" not in skip:
        def host(name):
            cols, types, chunks = side[name]
            return E.GpuHostBatchSource([[(dt, s, ch[c], None) for c, (dt, s) in zip(cols, types)] for ch in chunks])

        m.sync()
        m.set_alloc_limit(m.device_bytes_in_use() + (512 << 20))
        try:
            try:
                E.GpuShuffledHashJoinExec([lk], [ok], 0, host("lineitem"), host("orders")).collect()
                single = "finished"
            except m.B2Error as e:
                single = "error %d" % e.code
            gc.collect()
            s0 = m.memory_stats()["spilled_bytes"]
            j = E.GpuShuffledHashJoinExec([lk], [ok], 0, host("lineitem"), host("orders"), target_bytes=64 << 20)
            dt, outs = timed(m, lambda: collect(j))
            spilled = m.memory_stats()["spilled_bytes"] - s0
            stats = j.sub_partition_stats
        finally:
            m.set_alloc_limit(0)
        same = None if ref is None else all(np.array_equal(a, b) for a, b in zip(_rows(outs, nout), ref))
        print(json.dumps({"case": "c", "sf": sf, "alloc_limit_headroom": 512 << 20, "single_batch": single, "target": 64 << 20,
                          "sub_partitioned_wall_ms_incl_d2h_of_output": round(dt, 1), "spilled_bytes": spilled, "stats": stats,
                          "identical_to_b": same, "gpu": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=37_500_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--skip", default="")
    a = ap.parse_args()
    skip = set(a.skip.split(",")) if a.skip else set()
    import spark_rapids_b200 as m
    m.init(0)
    info = gpu_info()
    if "a" not in skip:
        bench_split(m, a.rows, a.reps, info)
    if not {"b", "c"} <= skip:
        bench_join(m, a.sf, a.reps, info, skip)


if __name__ == "__main__":
    main()
