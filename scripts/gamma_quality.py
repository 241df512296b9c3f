"""No GPU: what the TV-L1 illumination term (`gamma`, SURVEY.md A.8) does to accuracy, computed with the CPU oracle's
building blocks and the gamma steps of tests/tvl1_restate.py.  AEE against the analytic ground-truth flow of synth.pair
for gamma 0, 0.1 and 1, on the pair as it is, with frame b brightened (b * gain + offset) and with a horizontal brightness
ramp across frame b (0 at the left edge, `--ramp` grey levels at the right).  Prints a table and one JSON line.

    python scripts/gamma_quality.py [--size 256] [--gain 1.1] [--offset 8] [--ramp 24] [--seeds 0 1]
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

GAMMAS = [0.0, 0.1, 1.0]


def _u8(x):
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--gain", type=float, default=1.1)
    ap.add_argument("--offset", type=float, default=8.0)
    ap.add_argument("--ramp", type=float, default=24.0)
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1])
    args = ap.parse_args()
    rows = []
    for seed in args.seeds:
        a, b, gt = synth.pair(args.size, args.size, seed)
        bf = b.astype(np.float64)
        ramp = np.linspace(0.0, args.ramp, args.size)[None, :]
        inputs = {"unchanged": b, "gain+offset": _u8(bf * args.gain + args.offset), "ramp": _u8(bf + ramp)}
        for kind, fb in inputs.items():
            for g in GAMMAS:
                flow, log, _ = T.tvl1_calc(a, fb, gamma=g)
                rows.append({"seed": seed, "input": kind, "gamma": g, "aee_px": round(float(synth.aee(flow, gt)), 4),
                             "iterations": int(log.sum())})
                print("seed %d %-12s gamma %-4g: AEE %.4f px, %d iterations" % (seed, kind, g, rows[-1]["aee_px"], rows[-1]["iterations"]))
    print(json.dumps({"size": args.size, "gain": args.gain, "offset": args.offset, "ramp": args.ramp, "rows": rows}))


if __name__ == "__main__":
    main()
