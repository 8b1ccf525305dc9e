"""The hash table against the direct table (join.cu) for the two filtered FK -> PK joins of the TPC-H q3 plan at the SF100
batch size, the shapes of scripts/join_emit_bench.py:

  lineitem  37.5 M rows, l_shipdate > 1995-03-15, on l_orderkey against 14.6 M distinct order keys in [0, 1.5e8)
            (bitmap 18.75 MB); out [l_orderkey, l_extendedprice, l_discount] ++ [o_orderdate, o_shippriority]
  orders    18.75 M rows, o_orderdate < 1995-03-15, on o_custkey against 3 M distinct customer keys in [0, 1.5e7)
            (bitmap 1.9 MB); out [o_orderkey, o_orderdate, o_shippriority], nothing from the build side

Arms, each with B2_JOIN_NO_DIRECT=1 (hash) and without (direct), alternated:
  join    GpuFilterExec + GpuShuffledHashJoinExec over 1 + `--batches` copies of the batch (the first goes through the maps and
          sets the output estimate, the others are emitted by the probe): ms per batch (CUDA events, profiler off), kernel ms
          per batch (profiler on, separate run), algorithmic bytes over kernel time; and the build (b2_join_build alone).
  sweep   the lineitem batch's filter + probe (maps) against build sides whose bitmap is about 2, 8, 16, 19 and 32 MB at the
          lineitem join's density (10.3 key values per build row); the probe keys are l_orderkey scaled into the key range.
  sparse  a build side whose keys span 200x its rows (no direct table): the build with and without the direct attempt.
One JSON line per measurement.  The card, its power limit and its SM clock are read in the same run.

  python scripts/direct_join_bench.py [--batches 4] [--reps 3] [--out FILE]
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


def set_layout(layout):
    if layout == "hash":
        os.environ["B2_JOIN_NO_DIRECT"] = "1"
    else:
        os.environ.pop("B2_JOIN_NO_DIRECT", None)


def timed(m, fn, reps):
    """(mean ms over reps calls by CUDA events, profiler off; {kernel: ms per call} from one more call, profiler on)"""
    fn()
    e0 = m.Event().record()
    for _ in range(reps):
        fn()
    e1 = m.Event().record()
    ms = e0.elapsed_ms(e1) / reps
    m.profile_enable(True)
    fn()
    prof = {k["name"]: round(k["ms"], 4) for k in m.profile_report()}
    m.profile_enable(False)
    return ms, prof


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
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
    lines = []

    def emit(line):
        line["gpu"] = gpu_info()
        print(json.dumps(line), flush=True)
        lines.append(line)

    joins = [
        # name, stream columns, key, predicate column, predicate, keep, stream_out, build rows, key domain, build payload columns
        ("lineitem", [li["l_orderkey"], li["l_extendedprice"], li["l_discount"], li["l_shipdate"]], 0, 3, lambda c: c > m.lit(D, m.DATE32),
         li["l_shipdate"] > D, [0, 1, 2], 14_600_000, rows["orders"], [(4, m.DATE32), (4, m.INT32)]),
        ("orders", [od["o_orderkey"], od["o_custkey"], od["o_orderdate"], od["o_shippriority"]], 1, 2, lambda c: c < m.lit(D, m.DATE32),
         od["o_orderdate"] < D, [0, 2, 3], 3_000_000, rows["customer"], []),
    ]
    li_key, li_date = li["l_orderkey"], li["l_shipdate"]
    del li, od
    # ---- join: the q3 batches, hash against direct ---------------------------------------------------------------------------
    for name, cols, key, pcol, mk_pred, keep, so, nbuild, domain, payload in joins:
        n = len(cols[0])
        dts = [m.DATE32 if i == pcol or (name == "orders" and i == 2) else None for i in range(len(cols))]
        batch = m.Table.from_columns([m.Column.from_numpy(c, dtype=dt) for c, dt in zip(cols, dts)])
        bkey = rng.permutation(np.sort(rng.choice(domain, nbuild, replace=False))).astype(np.int64)
        bcols = [m.Column.from_numpy(bkey)] + [m.Column.from_numpy(rng.integers(0, 1 << 30, nbuild).astype(np.int32), dtype=dt) for _, dt in payload]
        build = m.Table.from_columns(bcols)
        keys_only = m.Table.from_columns([bcols[0]])
        bo = list(range(1, 1 + len(payload)))
        passing = np.flatnonzero(keep)
        hit = passing[np.isin(cols[key][passing], bkey)]
        matches = len(hit)
        widths = [cols[c].dtype.itemsize for c in so]
        out_bytes = matches * (sum(widths) + sum(w for w, _ in payload))
        stream_reads = sum(sectors(hit, w) for c, w in zip(so, widths) if c != key)
        pred_bytes = n * 4
        key_bytes = sectors(passing, 8)
        bpos = rng.integers(0, nbuild, matches)   # build rows hit: uniform, as the generator draws foreign keys
        span = int(bkey.max() - bkey.min() + 1)
        # HBM bytes of the table per layout: the Bloom filter, the bitmap and the block ranks are L2 residents (16 MB, <= 21 MB);
        # the hash layout reads one 16-byte slot (a 32-byte sector) per match, both read the payload row's sector per match
        pay = sectors(bpos, 8) if payload else 0
        table_bytes = {"hash": matches * 32 + pay, "direct": pay}
        pred = m.Program([mk_pred(m.col(pcol, m.DATE32, nullable=False))])
        for rep in range(args.reps):
            for layout in ("hash", "direct"):
                set_layout(layout)
                bms, bprof = timed(m, lambda: m.JoinHashTable(keys_only), 2)

                def plan():
                    flt = E.GpuFilterExec(pred, E.GpuBatchSource([batch] * (1 + args.batches)))
                    return E.GpuShuffledHashJoinExec([key], [0], m.JOIN_INNER, flt, E.GpuBatchSource([build]), stream_out=so, build_out=bo)
                list(plan())   # warm-up
                j = plan()
                it = iter(j)
                first = next(it)
                assert first.num_rows == matches, (name, first.num_rows, matches)
                del first
                e0 = m.Event().record()
                for t in it:
                    assert t.num_rows == matches
                    del t
                e1 = m.Event().record()
                ms = e0.elapsed_ms(e1) / args.batches
                stats = j.emit_stats
                j = plan()
                it = iter(j)
                next(it)
                m.profile_enable(True)
                for t in it:
                    del t
                prof = {k["name"]: round(k["ms"] / args.batches, 4) for k in m.profile_report()}
                m.profile_enable(False)
                kern = sum(prof.values())
                alg = pred_bytes + key_bytes + table_bytes[layout] + stream_reads + out_bytes
                emit({"arm": "join", "join": name, "layout": layout, "rep": rep, "stream_rows": n, "passing_rows": len(passing), "matches": matches,
                      "build_rows": nbuild, "key_span": span, "ms_per_batch": round(ms, 4), "kernel_ms_per_batch": prof,
                      "kernel_ms_sum": round(kern, 4), "emit_stats": stats, "build_ms": round(bms, 4), "build_kernels_ms": bprof,
                      "alg_bytes": int(alg), "alg_GBps_over_kernels": round(alg / 1e9 / (kern / 1e3), 1),
                      "frac_of_3350_GBps": round(alg / 1e9 / (kern / 1e3) / HBM_GBS, 3)})
        os.environ.pop("B2_JOIN_NO_DIRECT", None)
        del batch, build, keys_only
    # ---- sweep: bitmap size against L2 ----------------------------------------------------------------------------------------
    n = len(li_key)
    stream_date = m.Column.from_numpy(li_date, dtype=m.DATE32)
    pred = m.Program([m.col(1, m.DATE32, nullable=False) > m.lit(D, m.DATE32)])
    for mb in (2, 8, 16, 19, 32):
        span = mb * 8 << 20
        bkey = rng.permutation(np.unique(rng.integers(0, span, int(span / 10.3))))   # distinct: about 5 % fewer than drawn
        nbuild = len(bkey)
        skey = (li_key.astype(np.int64) * span // int(rows["orders"])).astype(np.int64)
        batch = m.Table.from_columns([m.Column.from_numpy(skey), stream_date])
        keys_only = m.Table.from_columns([m.Column.from_numpy(bkey)])
        for rep in range(args.reps):
            for layout in ("hash", "direct"):
                set_layout(layout)
                ht = m.JoinHashTable(keys_only)
                ms, prof = timed(m, lambda: ht.probe_filter(batch, 0, pred), 5)
                emit({"arm": "sweep", "bitmap_MB": round(span / 8 / 2**20, 2), "build_rows": nbuild, "layout": layout, "rep": rep,
                      "ms_per_probe": round(ms, 4), "kernel_ms": prof})
                del ht
        del batch, keys_only
    # ---- sparse: the cost of the attempt when the gate says no ----------------------------------------------------------------
    bkey = rng.permutation(np.unique(rng.integers(0, 200 * 14_600_000, 14_600_000)))
    nbuild = len(bkey)
    keys_only = m.Table.from_columns([m.Column.from_numpy(bkey)])
    for rep in range(args.reps):
        for layout in ("hash", "direct"):
            set_layout(layout)
            ms, prof = timed(m, lambda: m.JoinHashTable(keys_only), 5)
            emit({"arm": "sparse", "build_rows": nbuild, "key_span": int(bkey.max() - bkey.min() + 1), "layout": layout, "rep": rep,
                  "build_ms": round(ms, 4), "kernel_ms": prof})
    os.environ.pop("B2_JOIN_NO_DIRECT", None)
    if args.out:
        with open(args.out, "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
