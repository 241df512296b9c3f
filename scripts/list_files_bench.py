"""A video list from `-if` JPEG frame folders to flow files: `ListRunner.run_videos` (decode, gray, flow and the encodes on the
GPU) against the host path the list runner offered before it (imdecode + cvtColor on every host core, `run_list` for the
quantised planes, cv2.imencode of every plane on every host core).  Clips: 340x256 q95 4:2:0 JPEG frames, 64 per clip; two
workers per GPU; TV-L1 and Farneback; one GPU and every GPU.  Arms alternate; each arm's best of the rounds is reported as
flows/s.  Prints the GPU name and power limit and one JSON line.

    python scripts/list_files_bench.py [--clips 24] [--rounds 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from denseflow_b200 import listrun, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def clips(n, frames=64, h=256, w=340):
    import cv2
    out = []
    for c in range(n):
        gray = synth.stream(h, w, frames, seed=100 + c)
        bgr = [np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8) for g in gray]
        out.append([cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for f in bgr])
    return out


def gpu_arm(r, videos, save_type):
    n_files = [0]

    def on_chunk(video, dev, first, last, files):
        n_files[0] += len(files)

    t0 = time.perf_counter()
    st = r.run_videos(videos, step=1, bound=20, save_type=save_type, jpeg_exact=1, chunk_flows=64, on_chunk=on_chunk)
    return time.perf_counter() - t0, st["flows"], n_files[0]


def host_arm(r, videos, pool):
    """imdecode + gray on the host, the GPU for the planes, cv2.imencode of both planes of every flow on the host"""
    import cv2

    def decode(b):
        return cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)

    t0 = time.perf_counter()
    gray = [list(pool.map(decode, v)) for v in videos]
    futures = []

    def on_chunk(clip, dev, first, last, qx, qy, flows):
        planes = [p.copy() for p in qx] + [p.copy() for p in qy]  # the views die when the callback returns
        futures.extend(pool.submit(cv2.imencode, ".jpg", p) for p in planes)

    st = r.run(gray, step=1, bound=20, chunk_flows=64, on_chunk=on_chunk)
    n_files = sum(1 for f in futures if f.result()[0])
    return time.perf_counter() - t0, st["flows"], n_files


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    name, power = card()
    cores = len(os.sched_getaffinity(0))
    cv2.setNumThreads(1)
    ngpu = torch.cuda.device_count()
    videos = clips(a.clips)
    res = {"card": name, "power_limit": power, "gpus": ngpu, "host_cores": cores, "clip": "340x256 q95 4:2:0 JPEG, 64 frames",
           "clips": a.clips, "workers_per_gpu": 2, "flows_per_s": {}}
    pool = ThreadPoolExecutor(cores)
    for alg in ("tvl1", "farn"):
        for g in sorted({1, ngpu}):
            devices = [d for d in range(g) for _ in range(2)]
            r = listrun.ListRunner(alg, devices, 340, 256)
            arms = {"gpu_jpg": lambda: gpu_arm(r, videos, "jpg"), "gpu_png": lambda: gpu_arm(r, videos, "png"),
                    "host_decode_encode_jpg": lambda: host_arm(r, videos, pool)}
            for fn in arms.values():  # warm-up: handles, rings, encoders
                fn()
            best = {k: 0.0 for k in arms}
            files = {}
            for _ in range(a.rounds):
                for k, fn in arms.items():
                    sec, flows, nf = fn()
                    best[k] = max(best[k], flows / sec)
                    files[k] = nf
            r.close()
            key = "%s_%dgpu" % (alg, g)
            res["flows_per_s"][key] = {k: round(v, 1) for k, v in best.items()}
            res["flows_per_s"][key]["gpu_jpg_over_host"] = round(best["gpu_jpg"] / best["host_decode_encode_jpg"], 2)
            res["flows_per_s"][key]["files"] = files
            print(key, res["flows_per_s"][key], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
