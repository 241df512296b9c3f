"""-st=png throughput on one GPU: imencode(".png") on the GPU against cv2 on every host core, and the PNG batch call against
the u8 (-st=jpg planes) batch call on the same seeded frames.  Arms alternate after a warm-up; each arm's best of the rounds
is reported.  Prints the result as one JSON line, and also writes it to --out when given.

    python scripts/png_bench.py [--rounds 3] [--out result.json]
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


def packed_images(e, h, w, n):
    """Packed images of engine flows: the images -st=png encodes."""
    import torch
    frames = synth.stream(h, w, n + 1, 3)
    flows = e.calc_batch(list(frames))
    return [e.flow_to_png_image_device(torch.from_numpy(f).cuda(), return_bounds=False)[0] for f in flows]


def timed(fn, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import cv2
    import torch
    name, power = card()
    cores = len(os.sched_getaffinity(0))
    res = {"card": name, "power_limit": power, "host_cores": cores, "cv2": cv2.__version__, "encode": {}, "batch": {}}

    # 1. single-image encode: GPU (one call per image, each ending with the file on the host) vs cv2 on every core
    for (w, h) in [(340, 256), (1920, 1080)]:
        e = d.create("tvl1", 0, w, h)
        imgs = packed_images(e, h, w, 8)
        host = [i.cpu().numpy() for i in imgs]
        for i, x in zip(imgs, host):
            assert e.encode_png_bgr_device(i) == cv2.imencode(".png", x)[1].tobytes()
        pool = ThreadPoolExecutor(cores)
        reps = 64 if w < 1000 else 16
        gpu, cpu = [], []
        for _ in range(a.rounds + 1):
            torch.cuda.synchronize()
            gpu.append(timed(lambda: [e.encode_png_bgr_device(i) for i in imgs], max(1, reps // 8)) / len(imgs))
            cpu.append(timed(lambda: list(pool.map(lambda x: cv2.imencode(".png", x), host * (cores // len(host) + 1))),
                             max(1, reps // 8)) / (len(host) * (cores // len(host) + 1)))
        pool.shutdown()
        res["encode"]["%dx%d" % (w, h)] = {"gpu_images_per_s": 1 / min(gpu[1:]), "cv2_all_cores_images_per_s": 1 / min(cpu[1:]),
                                           "png_bytes_mean": float(np.mean([len(e.encode_png_bgr_device(i)) for i in imgs]))}
        e.release()

    # 2. the batch calls: flow -> PNG files vs flow -> quantised u8 planes (what the jpg branch encodes), same frames
    for alg, (w, h), n in [("tvl1", (1920, 1080), 22), ("tvl1", (340, 256), 130), ("farn", (340, 256), 130)]:
        e = d.create(alg, 0, w, h)
        frames = list(synth.stream(h, w, n, 9))
        m = n - 1
        cap = e._L.dfb_png_max_bytes(w, h)
        outs = [torch.empty(cap, dtype=torch.uint8, pin_memory=True).numpy() for _ in range(m)]
        qx = torch.empty((m, h, w), dtype=torch.uint8, pin_memory=True).numpy()
        qy = torch.empty((m, h, w), dtype=torch.uint8, pin_memory=True).numpy()
        e.calc_batch_png(frames, out=outs)
        e.calc_batch_u8_into(frames, 1, 20, qx, qy)
        tp, tu = [], []
        for _ in range(a.rounds):
            tp.append(timed(lambda: e.calc_batch_png(frames, out=outs), 1))
            tu.append(timed(lambda: e.calc_batch_u8_into(frames, 1, 20, qx, qy), 1))
        png_rate, u8_rate = m / min(tp), m / min(tu)
        res["batch"]["%s %dx%d" % (alg, w, h)] = {"pairs": m, "png_pairs_per_s": png_rate, "u8_pairs_per_s": u8_rate,
                                                 "png_over_u8": png_rate / u8_rate}
        e.release()

    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
