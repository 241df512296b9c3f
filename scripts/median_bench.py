"""TV-L1 with the optional median filtering of the flow (`median_filtering`, `median_interval`; DESIGN §4.3): pairs/s of
dfb_calc_batch_host at 1920x1080 and 340x256 with the median off, at window 3 and 5, every 30 and every 300 iterations,
and the inner iterations the pairs executed (the median changes when the convergence checks stop a warp).  Configurations
alternate after a warm-up; each one's best round is reported.  Prints the GPU name and power limit with the figures, as
one JSON line, and also writes it to --out when given.

    python scripts/median_bench.py [--rounds 3] [--out result.json]
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

import denseflow_b200 as d  # noqa: E402
from denseflow_b200 import synth  # noqa: E402

SIZES = [(1920, 1080, 16), (340, 256, 64)]  # w, h, frames per call (15 and 63 pairs)
CONFIGS = [(0, 30), (3, 30), (5, 30), (3, 300), (5, 300)]  # (median_filtering, median_interval); interval 300 = once per warp


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    name, power = card()
    rows = []
    for w, h, n in SIZES:
        frames = list(synth.stream(h, w, n, seed=1))
        e = d.OpticalFlowDual_TVL1.create(0, w, h)
        flows = np.empty((n - 1, h, w, 2), np.float32)
        best = {c: float("inf") for c in CONFIGS}
        iters = {}
        for r in range(args.rounds + 1):  # round 0 warms every configuration up
            for c in CONFIGS:
                e.set("median_filtering", c[0]).set("median_interval", c[1])
                t0 = time.perf_counter()
                e.calc_batch(frames, step=1, flows=flows)
                dt = time.perf_counter() - t0
                if r > 0:
                    best[c] = min(best[c], dt)
                else:
                    iters[c] = float(np.mean([e.tvl1_pair_stats(j).sum() for j in range(n - 1)]))
        e.release()
        for c in CONFIGS:
            rows.append({"size": "%dx%d" % (w, h), "median_filtering": c[0], "median_interval": c[1], "pairs": n - 1,
                         "pairs_per_s": round((n - 1) / best[c], 1), "iterations_per_pair": round(iters[c], 1)})
            print("%-9s median %d every %3d: %8.1f pairs/s, %7.1f inner iterations per pair" % (rows[-1]["size"], c[0], c[1],
                                                                                                   rows[-1]["pairs_per_s"], iters[c]))
    line = json.dumps({"gpu": name, "power_limit": power, "rounds": args.rounds, "rows": rows})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
