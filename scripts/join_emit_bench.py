"""Maps + gather against the emitting probe, for the two filtered FK -> PK joins of the TPC-H q3 plan at the SF100 batch size.

  lineitem  37.5 M rows (benchdata.tpch.q3_chunk, chunk 0), l_shipdate > 1995-03-15, on l_orderkey against 14.6 M distinct
            order keys; out [l_orderkey, l_extendedprice, l_discount] ++ [o_orderdate, o_shippriority] (8-byte payload)
  orders    18.75 M rows, o_orderdate < 1995-03-15, on o_custkey against 3 M distinct customer keys;
            out [o_orderkey, o_orderdate, o_shippriority], nothing from the build side
Each join is a GpuFilterExec + GpuShuffledHashJoinExec over 1 + `--batches` copies of the batch: the first copy goes through
the maps (it sets the output estimate), the others are timed, with B2_JOIN_NO_EMIT set (maps + gather_fixed_kernel) and
without (the emitting join_filter_probe_kernel).  One JSON line per (join, path): ms per batch (CUDA events over the timed
batches, profiler off), per-kernel ms per batch (profiler on, separate run), the HBM bytes each path needs (computed from the
data: 32-byte sectors of the random reads, maps written and read, output written) and their rate against the 3.35 TB/s H100
SXM data sheet.  The card, its power limit and its SM clock are read in the same run.

  python scripts/join_emit_bench.py [--batches 4] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0     # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def sectors(rows, width):
    return int(np.unique(rows.astype(np.int64) * width // 32).size) * 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import spark_rapids_b200 as m
    from benchdata import tpch
    from spark_rapids_b200 import execs as E
    m.init(0)
    rng = np.random.default_rng(5)
    D = tpch.Q3_DATE
    rows = tpch.q3_rows(100)
    li = tpch.q3_chunk("lineitem", 100, 0)
    od = tpch.q3_chunk("orders", 100, 0)
    joins = [
        # name, stream columns, key, predicate column, predicate, keep, stream_out, build rows, key domain, build payload columns
        ("lineitem", [li["l_orderkey"], li["l_extendedprice"], li["l_discount"], li["l_shipdate"]], 0, 3, lambda c: c > m.lit(D, m.DATE32),
         li["l_shipdate"] > D, [0, 1, 2], 14_600_000, rows["orders"], [(4, m.DATE32), (4, m.INT32)]),
        ("orders", [od["o_orderkey"], od["o_custkey"], od["o_orderdate"], od["o_shippriority"]], 1, 2, lambda c: c < m.lit(D, m.DATE32),
         od["o_orderdate"] < D, [0, 2, 3], 3_000_000, rows["customer"], []),
    ]
    del li, od
    lines = []
    for name, cols, key, pcol, mk_pred, keep, so, nbuild, domain, payload in joins:
        n = len(cols[0])
        dts = [m.DATE32 if i == pcol or (name == "orders" and i == 2) else None for i in range(len(cols))]
        batch = m.Table.from_columns([m.Column.from_numpy(c, dtype=dt) for c, dt in zip(cols, dts)])
        bkey = rng.permutation(np.sort(rng.choice(domain, nbuild, replace=False))).astype(np.int64)
        bcols = [m.Column.from_numpy(bkey)] + [m.Column.from_numpy(rng.integers(0, 1 << 30, nbuild).astype(np.int32), dtype=dt) for _, dt in payload]
        build = m.Table.from_columns(bcols)
        bo = list(range(1, 1 + len(payload)))
        passing = np.flatnonzero(keep)
        hit = passing[np.isin(cols[key][passing], bkey)]
        matches = len(hit)
        widths = [cols[c].dtype.itemsize for c in so]
        out_bytes = matches * (sum(widths) + sum(w for w, _ in payload))
        stream_reads = sum(sectors(hit, w) for c, w in zip(so, widths) if c != key)
        bpos = rng.integers(0, nbuild, matches)   # build rows hit: uniform, as the generator draws foreign keys
        bytes_maps = matches * 8 * 2 + sum(sectors(hit, w) for w in widths) + sum(sectors(bpos, w) for w, _ in payload) + out_bytes
        bytes_emit = stream_reads + (sectors(bpos, 8) if payload else 0) + out_bytes
        pred = m.Program([mk_pred(m.col(pcol, m.DATE32, nullable=False))])
        for path, env in (("maps_gather", "1"), ("emit", None)):
            if env:
                os.environ["B2_JOIN_NO_EMIT"] = env
            else:
                os.environ.pop("B2_JOIN_NO_EMIT", None)

            def plan():
                flt = E.GpuFilterExec(pred, E.GpuBatchSource([batch] * (1 + args.batches)))
                return E.GpuShuffledHashJoinExec([key], [0], m.JOIN_INNER, flt, E.GpuBatchSource([build]), stream_out=so, build_out=bo)
            for _ in range(2):   # warm-up
                j = plan()
                list(j)
            j = plan()
            it = iter(j)
            first = next(it)
            assert first.num_rows == matches, (name, first.num_rows, matches)
            del first
            e0 = m.Event().record()
            outs = 0
            for t in it:
                outs += 1
                assert t.num_rows == matches
                del t
            e1 = m.Event().record()
            ms = e0.elapsed_ms(e1) / args.batches
            stats = j.emit_stats
            info = gpu_info()
            j = plan()
            it = iter(j)
            next(it)
            m.profile_enable(True)
            for t in it:
                del t
            prof = {k["name"]: round(k["ms"] / args.batches, 4) for k in m.profile_report()}
            m.profile_enable(False)
            kern = sum(prof.values())
            alg = bytes_maps if path == "maps_gather" else bytes_emit
            line = {"join": name, "path": path, "stream_rows": n, "passing_rows": len(passing), "matches": matches, "build_rows": nbuild,
                    "ms_per_batch": round(ms, 4), "kernel_ms_per_batch": prof, "kernel_ms_sum": round(kern, 4), "emit_stats": stats,
                    "alg_hbm_bytes": int(alg), "alg_GBps_over_kernels": round(alg / 1e9 / (kern / 1e3), 1),
                    "frac_of_3350_GBps": round(alg / 1e9 / (kern / 1e3) / HBM_GBS, 3), "gpu": info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        os.environ.pop("B2_JOIN_NO_EMIT", None)
        del batch, build
    if args.out:
        with open(args.out, "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
