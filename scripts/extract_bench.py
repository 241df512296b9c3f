"""Frame-extraction mode (`-s=0`) throughput: one batch of 512 synthetic coloured 1920 x 1080 frames (the reference's
batch_maxsize), resized to 340 x 256 or kept as they are, then JPEG-encoded at quality 95.

  GPU arm: dfb_extract_frames_host on page-locked frames, a host clock around the blocking call, after a warm-up batch.
  CPU arm: cv2.resize + cv2.imencode(".jpg"), one frame per core in a process pool (OpenCV single-threaded per process),
           which is what extract_frames_video does per frame on the host.

64 distinct frames (synth.stream, coloured as tests/test_pipeline_gpu.py does) are cycled through the 512 frame pointers;
each frame is still uploaded, converted and encoded on its own.  Prints the GPU name and power limit (read-only
nvidia-smi query) and one JSON line.

    python scripts/extract_bench.py [--frames 512] [--reps 3]
"""
import argparse
import ctypes as C
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

W, H, UNIQUE, SEED = 1920, 1080, 64, 41
CASES = {"340x256": (340, 256), "no_resize": None}


def make_frames():
    from denseflow_b200 import synth
    gray = synth.stream(H, W, UNIQUE, seed=SEED)
    rng = np.random.default_rng(0)
    return np.stack([np.stack([np.roll(g, 3, 1), g, 255 - np.roll(g, 5, 0)], -1).astype(np.uint8)
                     ^ rng.integers(0, 4, g.shape + (3,), dtype=np.uint8) for g in gray])


def usable_cores():
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(per) + 0.5)))
    except Exception:
        pass
    return max(1, n)


_FRAMES = _SHM = None


def _cpu_init(shm_name, shape):
    """attach to the frames in shared memory (spawned workers: no copy per process, no OpenCV state inherited by fork)"""
    global _FRAMES, _SHM
    from multiprocessing import shared_memory
    import cv2
    cv2.setNumThreads(1)
    _SHM = shared_memory.SharedMemory(name=shm_name)
    _FRAMES = np.ndarray(shape, np.uint8, buffer=_SHM.buf)


def _cpu_frame(job):
    import cv2
    i, dst = job
    f = _FRAMES[i % len(_FRAMES)]
    if dst:
        f = cv2.resize(f, dst)
    ok, buf = cv2.imencode(".jpg", f)
    return len(buf)


def cpu_arm(frames, n, dst, reps):
    """frames/s of resize + imencode over all usable cores, one frame per task"""
    from multiprocessing import shared_memory
    cores = usable_cores()
    shm = shared_memory.SharedMemory(create=True, size=frames.nbytes)
    np.ndarray(frames.shape, np.uint8, buffer=shm.buf)[...] = frames
    pool = mp.get_context("spawn").Pool(cores, _cpu_init, (shm.name, frames.shape))
    try:
        pool.map(_cpu_frame, [(i, dst) for i in range(cores)])
        times = []
        for _ in range(reps):
            t0 = time.perf_counter()
            pool.map(_cpu_frame, [(i, dst) for i in range(n)], chunksize=1)
            times.append(time.perf_counter() - t0)
    finally:
        pool.close()
        pool.join()
        shm.close()
        shm.unlink()
    return {"frames_per_s": n / statistics.median(times), "runs_s": times, "cores": cores}


def gpu_arm(frames, n, dst, reps):
    import torch
    import denseflow_b200 as d
    e = d.create("farn", 0, W, H)
    pinned = torch.empty(frames.shape, dtype=torch.uint8, pin_memory=True)
    pinned.numpy()[...] = frames
    ptrs = [pinned[i % len(frames)].data_ptr() for i in range(n)]
    dw, dh = dst if dst else (0, 0)
    cap = e._L.dfb_jpeg_max_bytes_bgr(*(dst if dst else (W, H)))
    outs = [np.zeros(cap, np.uint8) for _ in range(n)]  # touched once, outside the timed region
    fp = (C.c_void_p * n)(*ptrs)
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    lens = (C.c_size_t * n)()

    def run():
        e._check(e._L.dfb_extract_frames_host(e._h, fp, n, W, H, dw, dh, 95, op, cap, lens))
    run()  # warm-up: allocations, encoder states, nvJPEG's own buffers
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        run()
        times.append(time.perf_counter() - t0)
    total = sum(lens)
    e.release()
    return {"frames_per_s": n / statistics.median(times), "runs_s": times, "mean_jpeg_bytes": total / n}


def gpu_name_and_power():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi failed: " + r.stderr.strip())
    return r.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    frames = make_frames()
    result = {"workload": "extract_frames_video batch: %d synthetic colour %dx%d frames, JPEG quality 95" % (args.frames, W, H),
              "frames": args.frames, "src": [W, H], "cases": {}}
    for name, dst in CASES.items():
        result["cases"][name] = {"cpu": cpu_arm(frames, args.frames, dst, args.reps)}
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device: the GPU arm cannot run")
    gpu = gpu_name_and_power()
    print("gpu:", gpu)
    result["gpu"] = gpu
    for name, dst in CASES.items():
        c = result["cases"][name]
        c["gpu"] = gpu_arm(frames, args.frames, dst, args.reps)
        c["speedup"] = c["gpu"]["frames_per_s"] / c["cpu"]["frames_per_s"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
