"""TV-L1 with the illumination term (`gamma`; SURVEY.md A.8, DESIGN §4.3): pairs/s of dfb_calc_batch_host at 1920x1080 and
340x256 with gamma off (0) and on (0.1 and 1.0), and the mean inner iterations per (scale, warp) the pairs executed.  The
clip's brightness drifts from frame to frame (gain and offset), the content the term is for.  Configurations alternate
after a warm-up; each one's best round is reported.  Prints the GPU name and power limit with the figures, as one JSON
line, and also writes it to --out when given.

    python scripts/gamma_bench.py [--rounds 3] [--out result.json]
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

SIZES = [(1920, 1080, 8), (340, 256, 64)]  # w, h, frames per call (7 and 63 pairs)
GAMMAS = [0.0, 0.1, 1.0]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def drifting(h, w, n):
    fr = synth.stream(h, w, n, seed=1).astype(np.float64)
    return [np.clip(np.rint(f * (1.0 + 0.01 * i) + 0.5 * i), 0, 255).astype(np.uint8) for i, f in enumerate(fr)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    name, power = card()
    rows = []
    for w, h, n in SIZES:
        frames = drifting(h, w, n)
        e = d.OpticalFlowDual_TVL1.create(0, w, h)
        flows = np.empty((n - 1, h, w, 2), np.float32)
        best = {g: float("inf") for g in GAMMAS}
        iters = {}
        for r in range(args.rounds + 1):  # round 0 warms every configuration up
            for g in GAMMAS:
                e.set("gamma", g)
                t0 = time.perf_counter()
                e.calc_batch(frames, step=1, flows=flows)
                dt = time.perf_counter() - t0
                if r > 0:
                    best[g] = min(best[g], dt)
                else:
                    logs = [e.tvl1_pair_stats(j) for j in range(n - 1)]
                    iters[g] = float(np.mean([lg[lg > 0].mean() for lg in logs]))
        e.release()
        for g in GAMMAS:
            rows.append({"size": "%dx%d" % (w, h), "gamma": g, "pairs": n - 1, "pairs_per_s": round((n - 1) / best[g], 1),
                         "iterations_per_scale_warp": round(iters[g], 1)})
            print("%-9s gamma %-4g: %8.1f pairs/s, %6.1f inner iterations per (scale, warp)" % (rows[-1]["size"], g, rows[-1]["pairs_per_s"],
                                                                                               iters[g]))
    line = json.dumps({"gpu": name, "power_limit": power, "rounds": args.rounds, "rows": rows})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
