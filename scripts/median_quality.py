"""No GPU: what the median filtering of the TV-L1 flow does to accuracy, computed with the CPU oracle's building blocks and
the median of tests/tvl1_restate.py.  AEE against the
analytic ground-truth flow of synth.pair, with the median off and at window 3 and 5 every 30 and every 300 iterations, on
the clean pair and on the same pair with salt-and-pepper pixels (each frame on its own, `--noise` of the pixels set to 0
or 255).  Prints a table and one JSON line.

    python scripts/median_quality.py [--size 256] [--noise 0.03] [--seeds 0 1]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tvl1_restate as T  # noqa: E402
from denseflow_b200 import synth  # noqa: E402

CONFIGS = [(0, 30), (3, 30), (5, 30), (3, 300), (5, 300)]


def salt_and_pepper(img, frac, rng):
    out = img.copy()
    hit = rng.random(img.shape) < frac
    out[hit] = np.where(rng.random(int(hit.sum())) < 0.5, 0, 255).astype(np.uint8)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--noise", type=float, default=0.03)
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1])
    args = ap.parse_args()
    rows = []
    for seed in args.seeds:
        a, b, gt = synth.pair(args.size, args.size, seed)
        rng = np.random.default_rng(1000 + seed)
        inputs = {"clean": (a, b), "salt-and-pepper": (salt_and_pepper(a, args.noise, rng), salt_and_pepper(b, args.noise, rng))}
        for kind, (fa, fb) in inputs.items():
            for k, interval in CONFIGS:
                flow, log, _ = T.tvl1_calc(fa, fb, median_filtering=k, median_interval=interval)
                rows.append({"seed": seed, "input": kind, "median_filtering": k, "median_interval": interval,
                             "aee_px": round(float(synth.aee(flow, gt)), 4), "iterations": int(log.sum())})
                print("seed %d %-15s median %d every %3d: AEE %.4f px, %d iterations" % (seed, kind, k, interval, rows[-1]["aee_px"],
                                                                                         rows[-1]["iterations"]))
    print(json.dumps({"size": args.size, "noise": args.noise, "rows": rows}))


if __name__ == "__main__":
    main()
