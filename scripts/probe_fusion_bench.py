"""Where the time of the filtered FK -> PK probe goes, on one q3-shaped batch at the SF100 batch size.

Two joins of the TPC-H q3 plan, one stream batch each (benchdata.tpch.q3_chunk, chunk 0):
  lineitem  37.5 M rows, l_shipdate > 1995-03-15 (~54 % pass), keyed on l_orderkey, against 14.6 M distinct order keys;
  orders    18.75 M rows, o_orderdate < 1995-03-15 (~49 % pass), keyed on o_custkey, against 3 M distinct customer keys.
The build keys are a uniform random subset of the key domain of the size q3's filtered build side has (the plan's own build
side is uniform too: the generator draws foreign keys uniformly).  Each join is timed through the C ABI as
  (a) b2_filter_row_ids + b2_join_probe_sel   the selection-vector path
  (b) b2_join_probe_filter                    the filter evaluated inside the probe (join_filter_probe_kernel)
  (c) (b) with a predicate no row passes      the streaming floor of the predicate column
  (d) (b) against disjoint build keys         streaming + Bloom lookups; only false positives reach the table
and prints one JSON line per (join, case): ms per call (CUDA events, profiler off), per-kernel ms (profiler on, separate
run), the HBM bytes the algorithm needs (computed from the data) and their rate against the 3.35 TB/s H100 SXM data sheet.
The card, its power limit and its SM clock are read in the same run.

  python scripts/probe_fusion_bench.py [--reps 20] [--out FILE]
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
    """bytes of the distinct 32-byte sectors that hold the given rows of a column of `width` bytes"""
    return int(np.unique(rows.astype(np.int64) * width // 32).size) * 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import spark_rapids_b200 as m
    from benchdata import tpch
    m.init(0)
    rng = np.random.default_rng(5)
    D = tpch.Q3_DATE
    rows = tpch.q3_rows(100)
    li = tpch.q3_chunk("lineitem", 100, 0)
    od = tpch.q3_chunk("orders", 100, 0)
    joins = [
        # name, key column, predicate column, predicate, a predicate nothing passes, build size, key domain
        ("lineitem", li["l_orderkey"], li["l_shipdate"], lambda c: c > m.lit(D, m.DATE32), li["l_shipdate"] > D, 14_600_000, rows["orders"]),
        ("orders", od["o_custkey"], od["o_orderdate"], lambda c: c < m.lit(D, m.DATE32), od["o_orderdate"] < D, 3_000_000, rows["customer"]),
    ]
    del li, od
    lines = []
    for name, key, date, mk_pred, keep, nbuild, domain in joins:
        n = len(key)
        table = m.Table.from_columns([m.Column.from_numpy(key), m.Column.from_numpy(date, dtype=m.DATE32)])
        keys_only = m.Table.from_columns([m.Column.from_numpy(key)])
        c = m.col(1, m.DATE32, nullable=False)
        pred = m.Program([mk_pred(c)])
        none = m.Program([c < m.lit(0, m.DATE32)])
        bkey = np.sort(rng.choice(domain, nbuild, replace=False)).astype(np.int64)
        ht = m.JoinHashTable(m.Table.from_columns([m.Column.from_numpy(bkey)]))
        ht_disjoint = m.JoinHashTable(m.Table.from_columns([m.Column.from_numpy(bkey + domain)]))
        passing = np.flatnonzero(keep)
        npass = len(passing)
        matches = int(np.isin(key[passing], bkey).sum())
        key_bytes = sectors(passing, 8)
        maps = matches * 8
        cases = {
            "a_selection_vector": (lambda: ht.probe(keys_only, m.JOIN_INNER, selection=m.filter_row_ids(pred, table)),
                                   n * 4 + npass * 4 + npass * 4 + key_bytes + maps, npass, matches),
            "b_fused": (lambda: ht.probe_filter(table, 0, pred), n * 4 + key_bytes + maps, npass, matches),
            "c_fused_none_pass": (lambda: ht.probe_filter(table, 0, none), n * 4, 0, 0),
            "d_fused_disjoint_build": (lambda: ht_disjoint.probe_filter(table, 0, pred), n * 4 + key_bytes, npass, 0),
        }
        for case, (fn, alg_bytes, bloom_lookups, want_matches) in cases.items():
            for _ in range(args.warmup):
                res = fn()
            assert len(res[0]) == want_matches, (name, case, len(res[0]), want_matches)
            del res
            ms = []
            for _ in range(args.reps):
                e0 = m.Event().record()
                res = fn()
                e1 = m.Event().record()
                ms.append(e0.elapsed_ms(e1))
                del res
            info = gpu_info()   # right after the timed loop: the SM clock under this load
            m.profile_enable(True)
            for _ in range(args.reps):
                res = fn()
                del res
            prof = {k["name"]: round(k["ms"] / args.reps, 4) for k in m.profile_report()}
            m.profile_enable(False)
            med = float(np.median(ms))
            kern = sum(prof.values())
            line = {"join": name, "case": case, "stream_rows": n, "passing_rows": bloom_lookups, "matches": want_matches, "build_rows": nbuild,
                    "ms_per_call_median": round(med, 4), "ms_per_call_min": round(min(ms), 4), "ms_per_call_max": round(max(ms), 4),
                    "kernel_ms_per_call": prof, "kernel_ms_sum": round(kern, 4),
                    "alg_hbm_bytes": int(alg_bytes), "alg_GBps_over_kernels": round(alg_bytes / 1e9 / (kern / 1e3), 1) if kern else None,
                    "frac_of_3350_GBps": round(alg_bytes / 1e9 / (kern / 1e3) / HBM_GBS, 3) if kern else None,
                    "bloom_lookups_L2": bloom_lookups, "gpu": info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        del table, keys_only, ht, ht_disjoint
    if args.out:
        with open(args.out, "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
