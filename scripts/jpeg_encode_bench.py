"""Exact JPEG encode throughput on one GPU (the "jpeg_exact" handle parameter and dfb_encode_jpeg_gray_batch_device):
gray images/s of the exact batch call, of nvJPEG one plane per call and of cv2.imencode on every host core; pairs/s of
dfb_process_bgr_batch_host and frames/s of dfb_extract_frames_host with jpeg_exact 1 against 0; the time of each encoder
kernel for one 3840x2160 colour frame (torch.profiler).  Every arm runs once as a warm-up, then the arms alternate for
--rounds rounds and each arm's best round is reported.  Prints the result as one JSON line, and also writes it to --out when given.

    python scripts/jpeg_encode_bench.py [--rounds 3] [--out result.json]
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

import denseflow_b200 as d  # noqa: E402
from denseflow_b200 import synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def best_rate(arms, rounds, count):
    """arms: {name: fn}; one warm-up call per arm, then every arm once per round, alternating; returns
    {name: count / best seconds}"""
    for fn in arms.values():
        fn()
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t0 = time.perf_counter()
            fn()
            t[k].append(time.perf_counter() - t0)
    return {k: count[k] / min(v) if isinstance(count, dict) else count / min(v) for k, v in t.items()}


def colour(gray):
    return [np.stack([np.roll(g, 3, 1), g, 255 - np.roll(g, 5, 0)], -1).astype(np.uint8) for g in gray]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    name, power = card()
    cores = len(os.sched_getaffinity(0))
    res = {"card": name, "power_limit": power, "host_cores": cores, "cv2": cv2.__version__, "gray_encode": {}, "chain": {}, "extract": {}}

    # 1. gray planes: exact batch vs nvJPEG one plane per call vs cv2 on every core (quantised flow planes of the engine)
    for (w, h, n) in [(1920, 1080, 16), (340, 256, 128)]:
        e = d.create("tvl1", 0, w, h)
        qx, qy = e.calc_batch(list(synth.stream(h, w, n // 2 + 1, 3)), step=1, bound=20)
        host = [p for pair in zip(qx, qy) for p in pair][:n]
        dev = torch.from_numpy(np.stack(host)).cuda()
        exact = e.encode_jpeg_gray_batch_device(dev, 95)
        assert exact == [cv2.imencode(".jpg", p, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for p in host]
        pool = ThreadPoolExecutor(cores)
        e.encode_jpeg_gray_device(dev[0], 95)
        r = best_rate({"exact_batch": lambda: e.encode_jpeg_gray_batch_device(dev, 95),
                       "nvjpeg_per_plane": lambda: [e.encode_jpeg_gray_device(dev[i], 95) for i in range(n)],
                       "cv2_all_cores": lambda: list(pool.map(lambda p: cv2.imencode(".jpg", p), host))}, a.rounds, n)
        pool.shutdown()
        res["gray_encode"]["%dx%d" % (w, h)] = {k + "_images_per_s": v for k, v in r.items()}
        e.release()

    # 2. dfb_process_bgr_batch_host, jpeg_exact 1 vs 0
    for (alg, w, h, n) in [("tvl1", 1920, 1080, 17), ("tvl1", 340, 256, 65), ("farn", 340, 256, 65)]:
        e = d.create(alg, 0, w, h)
        bgr = colour(synth.stream(h, w, n, 5))

        def run(x, e=e, bgr=bgr):
            e.set("jpeg_exact", x)
            e.process_bgr_batch(bgr, step=1, bound=20)
        run(0)
        run(1)
        r = best_rate({"nvjpeg": lambda: run(0), "exact": lambda: run(1)}, a.rounds, n - 1)
        res["chain"]["%s_%dx%d" % (alg, w, h)] = {"nvjpeg_pairs_per_s": r["nvjpeg"], "exact_pairs_per_s": r["exact"],
                                                  "ratio": r["exact"] / r["nvjpeg"]}
        e.release()

    # 4. per-kernel device time of one 3840x2160 colour frame (the single-CTA scans are the stages that do not fill the GPU)
    from torch.profiler import ProfilerActivity, profile
    e = d.create("farn", 0, 3840, 2160)
    e.set("jpeg_exact", 1)
    frame = torch.from_numpy(colour(synth.stream(2160, 3840, 1, 7))[0]).cuda()
    e.encode_jpeg_bgr_device(frame)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            e.encode_jpeg_bgr_device(frame)
    stages = {}
    for ev in prof.key_averages():
        if "k_" in ev.key and ev.count:
            k = ev.key.split("k_", 1)[1].split("(")[0].split("<")[0]
            stages["k_" + k] = ev.device_time_total / ev.count if hasattr(ev, "device_time_total") else ev.cuda_time_total / ev.count
    res["stages_3840x2160_bgr_us"] = stages
    e.release()

    # 3. dfb_extract_frames_host, jpeg_exact 1 vs 0
    e = d.create("farn", 0, 1920, 1080)
    frames = colour(synth.stream(1080, 1920, 32, 6))
    for dst in [(340, 256), None]:
        def run(x, dst=dst):
            e.set("jpeg_exact", x)
            e.extract_frames(frames, dst, 95)
        run(0)
        run(1)
        r = best_rate({"nvjpeg": lambda: run(0), "exact": lambda: run(1)}, a.rounds, len(frames))
        res["extract"]["1920x1080->" + ("%dx%d" % dst if dst else "same")] = {"nvjpeg_frames_per_s": r["nvjpeg"], "exact_frames_per_s": r["exact"],
                                                                            "ratio": r["exact"] / r["nvjpeg"]}
    e.release()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
