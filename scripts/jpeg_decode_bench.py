"""Throughput of the imdecode-exact GPU JPEG decoder (dfb_decode_jpeg_batch_device) and of the `-if` flow chain built on it.

Gray frames/s for q95 4:2:0 colour frames at 340x256 and 1920x1080:
  gpu_exact   decode_jpeg_batch(channels=1), batches of 32 files
  nvjpeg      dfb_decode_jpeg_gray_device, one file per call (not bit-exact)
  cv2         imdecode + cvtColor on every usable host core (thread pool)
Chain pairs/s: process_jpeg_batch (JPEG files in) against process_bgr_batch (pinned BGR frames in): TV-L1 at 1080p and
340x256, Farneback at 340x256.  Best of --reps runs, variants alternated.  Prints one JSON line (--out FILE also writes it),
with the card name and power limit read in the same run, and the sync rounds the decoder took.
    python scripts/jpeg_decode_bench.py [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20).stdout.strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception:
        return ["unknown", "unknown"]


def frames(n, h, w):
    from denseflow_b200 import synth
    gray = synth.stream(h, w, n, seed=3)
    bgr = [np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8) for g in gray]
    return bgr, [cv2.imencode(".jpg", b, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for b in bgr]


def usable_cores():
    return len(os.sched_getaffinity(0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import denseflow_b200 as d
    name, plimit = card()
    res = {"card": name, "power_limit": plimit, "host_cores": usable_cores(), "decode_frames_per_s": {}, "chain_pairs_per_s": {},
           "sync_rounds": {}}
    pool = ThreadPoolExecutor(usable_cores())
    for (w, h) in [(340, 256), (1920, 1080)]:
        bgr, jpgs = frames(32, h, w)
        e = d.create("farn", 0, w, h)
        res["sync_rounds"]["%dx%d" % (w, h)] = e.debug_jpeg_coefficients(jpgs[0])[1]
        dev = torch.empty((h, w), dtype=torch.uint8, device="cuda")
        best = {"gpu_exact": 0.0, "nvjpeg": 0.0, "cv2": 0.0}
        e.decode_jpeg_batch(jpgs, 1)
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            e.decode_jpeg_batch(jpgs, 1)
            torch.cuda.synchronize()
            best["gpu_exact"] = max(best["gpu_exact"], len(jpgs) / (time.perf_counter() - t))
            t = time.perf_counter()
            for j in jpgs:
                e.decode_jpeg_gray_device(j, w, h)
            torch.cuda.synchronize()
            best["nvjpeg"] = max(best["nvjpeg"], len(jpgs) / (time.perf_counter() - t))
            t = time.perf_counter()
            list(pool.map(lambda j: cv2.cvtColor(cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY), jpgs))
            best["cv2"] = max(best["cv2"], len(jpgs) / (time.perf_counter() - t))
        res["decode_frames_per_s"]["%dx%d" % (w, h)] = {k: round(v, 1) for k, v in best.items()}
    for alg, (w, h), n in [("tvl1", (1920, 1080), 17), ("tvl1", (340, 256), 65), ("farn", (340, 256), 65)]:
        bgr, jpgs = frames(n, h, w)
        pinned = []
        for b in bgr:
            t = torch.empty(b.shape, dtype=torch.uint8).pin_memory()
            t.numpy()[:] = b
            pinned.append(t.numpy())
        e = d.create(alg, 0, w, h)
        e.process_jpeg_batch(jpgs[:3], 1, 20)
        e.process_bgr_batch(pinned[:3], 1, 20)
        best = {"jpeg": 0.0, "bgr": 0.0}
        for _ in range(args.reps):
            t = time.perf_counter()
            e.process_jpeg_batch(jpgs, 1, 20)
            best["jpeg"] = max(best["jpeg"], (n - 1) / (time.perf_counter() - t))
            t = time.perf_counter()
            e.process_bgr_batch(pinned, 1, 20)
            best["bgr"] = max(best["bgr"], (n - 1) / (time.perf_counter() - t))
        best = {k: round(v, 1) for k, v in best.items()}
        best["ratio"] = round(best["jpeg"] / best["bgr"], 3)
        res["chain_pairs_per_s"]["%s %dx%d" % (alg, w, h)] = best
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
