"""What an outer join that preserves the build side costs, on TPC-H q13's shape: customer LEFT OUTER JOIN orders ON
c_custkey = o_custkey AND <predicate on orders>, then a count of orders per customer.  The q3 generator (benchdata.tpch) has
no o_comment, so the predicate is o_orderdate < 1997-01-01 (about 70 % of the orders) in place of q13's comment LIKE.

  (a) today's plan: LEFT OUTER, stream customer, build the filtered orders (a non-distinct build side: the generic probe);
  (b) RIGHT OUTER (= LeftOuter / BuildLeft with the children swapped): build customer, stream orders, the filter fused into
      the probe (join_filter_probe_track_kernel), the unmatched customers emitted at the end (tracker_count / tracker_write);
  (c) the probe of (b) as INNER against RIGHT OUTER: the cost of tracking;
  (d) (b) as FULL OUTER without a condition: the filtered orders probe LEFT OUTER, tracked, one stream batch at a time.

Every arm runs the GpuShuffledHashJoinExec over device-resident batches (8 chunks per table).  Reported per arm: wall ms
(host clock around the whole join and a device synchronise, profiler off, the arms alternated, median of --reps), per-kernel
ms from a separate profiled call, the bytes the probe and tracker kernels need (below) over their kernel time against the
3.35 TB/s H100 SXM data sheet, and count(*) per c_custkey, checked equal between (a) and (b) and, for the rows of (d) that
carry a customer, between (b) and (d); (d) also reports its output rows.  The card and its power limit
are read in the same run.  One JSON line per measurement.
  filter probe:     4 B o_orderdate per order, 8 B o_custkey + one 16-byte table slot per passing order, 8 B of maps per pair
  tracker kernels:  nb / 8 bytes of bitmap read twice, 4 B per unmatched customer written

  python scripts/build_side_outer_join_bench.py [--sf 10 | --sf 100] [--reps 3]
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
DATE_1997_01_01 = 9862


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import spark_rapids_b200 as m
    from spark_rapids_b200 import execs as E
    from benchdata import tpch
    m.init(0)
    info = gpu_info()
    cust, orders = [], []
    for i in range(tpch.Q3_CHUNKS["customer"]):
        c = tpch.q3_chunk("customer", args.sf, i)
        cust.append(m.Table.from_columns([m.Column.from_numpy(c["c_custkey"])]))
    for i in range(tpch.Q3_CHUNKS["orders"]):
        o = tpch.q3_chunk("orders", args.sf, i)
        orders.append(m.Table.from_columns([m.Column.from_numpy(o["o_orderkey"]), m.Column.from_numpy(o["o_custkey"]),
                                            m.Column.from_numpy(o["o_orderdate"], dtype=m.DATE32)]))
    ncust = sum(t.num_rows for t in cust)
    nord = sum(t.num_rows for t in orders)
    pred = m.Program([m.col(2, m.DATE32, nullable=False) < m.lit(DATE_1997_01_01, m.DATE32)])

    def plan(arm):
        filtered = E.GpuFilterExec(pred, E.GpuBatchSource(orders))
        if arm == "a":   # stream customer, build the filtered orders; out: c_custkey, o_orderkey
            return E.GpuShuffledHashJoinExec([0], [1], m.JOIN_LEFT_OUTER, E.GpuBatchSource(cust), filtered, stream_out=[0], build_out=[0])
        kind = {"b": m.JOIN_RIGHT_OUTER, "c": m.JOIN_INNER, "d": m.JOIN_FULL_OUTER}[arm]   # stream the filtered orders, build customer; out: o_orderkey, c_custkey
        return E.GpuShuffledHashJoinExec([1], [0], kind, filtered, E.GpuBatchSource(cust), stream_out=[0], build_out=[0])

    def run(arm, keep=False):
        j = plan(arm)
        outs = list(j)
        m.sync()
        if not keep:
            del outs
            return None
        return outs

    def counts(arm, outs, without_customer=None):
        ck, ok = (0, 1) if arm == "a" else (1, 0)
        cnt = np.zeros(ncust, np.int64)
        rows = np.zeros(ncust, np.int64)
        for t in outs:
            c, cv = t.column(ck).to_numpy()
            _, ov = t.column(ok).to_numpy()
            if without_customer is None:
                assert cv.all()
            else:   # FULL OUTER: orders without a customer keep a NULL c_custkey
                without_customer.append(int((~cv).sum()))
                c, ov = c[cv], ov[cv]
            np.add.at(rows, c, 1)
            np.add.at(cnt, c[ov], 1)
        return cnt, rows

    # correctness: count(*) per customer, (a) against (b)
    ca, ra = counts("a", run("a", True))
    cb, rb = counts("b", run("b", True))
    assert np.array_equal(ca, cb), "count per c_custkey differs between (a) and (b)"
    assert (rb >= 1).all() and (ra >= 1).all()
    unmatched = int((cb == 0).sum())
    outs_d = run("d", True)
    nd = []
    cd, rd = counts("d", outs_d, nd)
    assert np.array_equal(cd, cb) and np.array_equal(rd, rb), "count per c_custkey differs between (b) and (d)"
    print(json.dumps({"check": "count(*) per c_custkey equal in (a) and (b), and in (b) and (d)", "sf": args.sf, "customers": ncust,
                      "orders": nord, "orders_passing": int(cb.sum()), "customers_without_orders": unmatched,
                      "full_outer_rows": sum(t.num_rows for t in outs_d), "full_outer_batches": len(outs_d),
                      "full_outer_rows_without_customer": sum(nd)}), flush=True)
    del outs_d
    gc.collect()

    # wall: arms alternated, profiler off
    walls = {a: [] for a in "abcd"}
    for a in "abcd":
        run(a)   # warm-up
    for _ in range(args.reps):
        for a in "abcd":
            m.sync()
            t0 = time.perf_counter()
            run(a)
            walls[a].append((time.perf_counter() - t0) * 1e3)
    # per-kernel ms, one profiled call per arm
    for a in "abcd":
        m.profile_enable(True)
        try:
            run(a)
            kern = {k["name"]: round(k["ms"], 3) for k in m.profile_report()}
        finally:
            m.profile_enable(False)
        npass = int(cb.sum())
        rec = {"arm": {"a": "left outer, build filtered orders", "b": "right outer, build customer, filter in probe",
                       "c": "inner, build customer, filter in probe", "d": "full outer, build customer, no condition"}[a],
               "sf": args.sf, "wall_ms": [round(x, 2) for x in walls[a]], "wall_ms_median": round(float(np.median(walls[a])), 2),
               "kernel_ms": kern, "gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_max": info.get("clocks.max.sm")}
        probe_k = "join_filter_probe_track_kernel" if a == "b" else "join_filter_probe_kernel"
        if a in "bc" and probe_k in kern:
            pb = 4 * nord + (8 + 16 + 8) * npass
            rec["probe_kernel"] = probe_k
            rec["probe_bytes"] = pb
            rec["probe_gbs"] = round(pb / (kern[probe_k] * 1e-3) / 1e9, 1)
            rec["probe_share_of_3.35TBs"] = round(pb / (kern[probe_k] * 1e-3) / 1e9 / HBM_GBS, 3)
        if a == "b":
            tb = 2 * ((ncust + 31) // 32) * 4 + 4 * unmatched
            tk = kern.get("tracker_count_kernel", 0) + kern.get("tracker_write_kernel", 0)
            rec["tracker_bytes"] = tb
            rec["tracker_kernel_ms"] = round(tk, 3)
            if tk:
                rec["tracker_gbs"] = round(tb / (tk * 1e-3) / 1e9, 1)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
