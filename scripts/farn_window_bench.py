"""Farneback's create() options `gaussian_window` (OPTFLOW_FARNEBACK_GAUSSIAN) and `fast_pyramids` (fastPyramids; SURVEY
B.7): pairs/s of dfb_calc_batch_device at 1280x720 and 340x256 for the four combinations, on device-resident synth.stream
frames and flows.  The four arms alternate after a warm-up round; each one's best of --rounds rounds is reported.  Prints
the GPU name and power limit, read in the same call, with the figures as one JSON line, and also writes it to --out when
given.

    python scripts/farn_window_bench.py [--rounds 3] [--out result.json]
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

SIZES = [(1280, 720, 33), (340, 256, 129)]  # w, h, frames per call (32 and 128 pairs)
ARMS = [(0, 0), (1, 0), (0, 1), (1, 1)]  # (gaussian_window, fast_pyramids)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    name, power = card()
    rows = []
    for w, h, n in SIZES:
        frames = torch.from_numpy(np.ascontiguousarray(synth.stream(h, w, n, seed=1))).cuda()
        flows = torch.empty((n - 1, h, w, 2), dtype=torch.float32, device="cuda")
        e = d.FarnebackOpticalFlow.create(0, w, h)
        best = {a: float("inf") for a in ARMS}
        for r in range(args.rounds + 1):  # round 0 warms every arm up
            for a in ARMS:
                e.set("gaussian_window", a[0]).set("fast_pyramids", a[1])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e.calc_batch_device(frames, step=1, flows=flows)
                torch.cuda.synchronize()
                if r > 0:
                    best[a] = min(best[a], time.perf_counter() - t0)
        e.release()
        for a in ARMS:
            rows.append({"size": "%dx%d" % (w, h), "gaussian_window": a[0], "fast_pyramids": a[1], "pairs": n - 1,
                         "pairs_per_s": round((n - 1) / best[a], 1)})
            print("%-9s gaussian_window %d fast_pyramids %d: %8.1f pairs/s" % (rows[-1]["size"], a[0], a[1], rows[-1]["pairs_per_s"]))
    line = json.dumps({"gpu": name, "power_limit": power, "rounds": args.rounds, "rows": rows})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
