"""Byte accounting of the radix group-by's materialise + first pass on a q3-shaped input (31.3 M rows of (INT64, DATE32, INT32)
keys, price and discount DECIMAL64, 12.9 M groups, SUM(price * (1 - disc)) as DECIMAL128), through the fused first pass and
through the separate one (B2_AGG_NO_FUSED_FIRST_PASS).  Prints per kernel the mean ms per call, the algorithmic bytes per
row and per call, the rate and its share of the 3.35 TB/s HBM3 data sheet.

Bytes per row (w = 36: h 4 + k0 8 + k1 8 + v 16; the join output it reads: 16 B of keys + 16 B of price and discount):
  part_tile_hist_kernel(keys)  16       the key columns
  radix_rows_scatter_kernel    32 + 36  keys, price, disc in; every materialised array out, in first-digit order
  radix_rows_kernel            32 + 36  the same arrays, in input order
  part_tile_hist_kernel        4        the hash array (one per scatter pass)
  part_scatter2_kernel         36 + 36  every array in and out
usage: python scripts/radix_fused_probe.py [rows] [groups] [reps]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import spark_rapids_b200 as m  # noqa: E402

PEAK = 3.35e12
W = 36
BYTES_PER_ROW = {"part_tile_hist_kernel(keys)": 16, "radix_rows_scatter_kernel": 32 + W, "radix_rows_kernel": 32 + W,
                 "part_tile_hist_kernel": 4, "part_scatter2_kernel": 2 * W}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 31_300_000
    g = int(sys.argv[2]) if len(sys.argv) > 2 else 12_900_000
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    m.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    rng = np.random.default_rng(3)
    k0 = (np.arange(n, dtype=np.int64) * 1_000_003) % g
    t = m.Table.from_columns([m.Column.from_numpy(k0), m.Column.from_numpy((8000 + k0 % 2557).astype(np.int32), dtype=m.DATE32),
                              m.Column.from_numpy((k0 % 5).astype(np.int32)),
                              m.Column.from_numpy(rng.integers(90_000, 10_494_951, n, dtype=np.int64), dtype=m.DECIMAL64, scale=2),
                              m.Column.from_numpy(rng.integers(0, 11, n, dtype=np.int64), dtype=m.DECIMAL64, scale=2)])
    one = m.lit(1, m.DECIMAL32, 1, 0)
    price, disc = m.col(3, m.DECIMAL64, 12, 2, nullable=False), m.col(4, m.DECIMAL64, 12, 2, nullable=False)
    prog = m.Program([m.col(0, m.INT64, nullable=False), m.col(1, m.DATE32, nullable=False), m.col(2, m.INT32, nullable=False),
                      price * (one - disc)])
    spec = [(m.AGG_SUM, 3, m.DECIMAL128, 4, 36)]
    for label, env in (("fused first pass", None), ("separate first pass", "1")):
        if env:
            os.environ["B2_AGG_NO_FUSED_FIRST_PASS"] = env
        else:
            os.environ.pop("B2_AGG_NO_FUSED_FIRST_PASS", None)
        m.scan_aggregate(prog, False, t, [0, 1, 2], spec)
        m.profile_enable(True)
        for _ in range(reps):
            m.scan_aggregate(prog, False, t, [0, 1, 2], spec)
        rep = m.profile_report()
        m.profile_enable(False)
        print("%s, %d rows, %d groups, %d calls:" % (label, n, g, reps))
        chain = 0.0
        for k in rep:
            ms = k["ms"] / reps
            per_call = k["launches"] / reps
            line = "  %-30s %7.3f ms per call (%g launches)" % (k["name"], ms, per_call)
            if k["name"] in BYTES_PER_ROW:
                b = BYTES_PER_ROW[k["name"]] * n * per_call
                chain += ms
                line += "  %5.2f GB  %5.2f TB/s  %.2f of the data sheet" % (b / 1e9, b / (ms * 1e-3) / 1e12, b / (ms * 1e-3) / PEAK)
            print(line)
        print("  materialise + scatter passes: %.3f ms per call" % chain)
    os.environ.pop("B2_AGG_NO_FUSED_FIRST_PASS", None)


if __name__ == "__main__":
    main()
