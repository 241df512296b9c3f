"""-st=h5 throughput on one GPU: pairs/s of dfb_calc_batch_host_planes (the two float planes the h5 datasets hold) against
dfb_calc_batch_host (the float2 field) and dfb_calc_batch_host_u8 (the -st=jpg planes) on the same seeded frames, TV-L1 at
1920x1080 and 340x256 with page-locked outputs; then the writer's MB/s for those planes to a tmpfs (/dev/shm) and to the
output directory's disk, and whether the D2H (planes call) or the file write bounds a 1080p chain.  Arms alternate after a
warm-up; each arm's best of the rounds is reported.  Prints one JSON line, and also writes it to --out when given.

    python scripts/h5_bench.py [--rounds 3] [--pairs 16] [--out result.json] [--disk DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import denseflow_b200 as d  # noqa: E402
from denseflow_b200 import h5, synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def pinned(shape, dtype):
    import torch
    return torch.empty(shape, dtype={np.float32: torch.float32, np.uint8: torch.uint8}[dtype], pin_memory=True).numpy()


def write_rate(planes, directory, rounds):
    """MB/s of writing every plane of `planes` [M,2,H,W] as the datasets of one h5 file in `directory` (best of the rounds)"""
    m = planes.shape[0]
    best = 0.0
    for _ in range(rounds):
        fd, path = tempfile.mkstemp(suffix=".h5", dir=directory)
        os.close(fd)
        t = time.perf_counter()
        with h5.File(path, variant="hdf5") as f:
            for c, tag in ((0, "x"), (1, "y")):
                for i in range(m):
                    f.write_float("/flow_%s_%05d" % (tag, i), planes[i, c])
        fdd = os.open(path, os.O_RDONLY)
        os.fsync(fdd)
        os.close(fdd)
        dt = time.perf_counter() - t
        best = max(best, planes.nbytes / dt / 1e6)
        os.unlink(path)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--disk", default=None, help="directory on disk for the writer's disk rate (default: a temporary directory)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    res = {"gpu": name, "power_limit": power, "pairs": a.pairs, "calls": {}, "writer_MBps": {}}
    planes_1080 = None
    for (w, h) in ((1920, 1080), (340, 256)):
        fr = synth.stream(h, w, a.pairs + 1, 7)
        m = a.pairs
        e = d.create("tvl1", 0, w, h, variant="hdf5")
        flows = pinned((m, h, w, 2), np.float32)
        planes = pinned((m, 2, h, w), np.float32)
        qx, qy = pinned((m, h, w), np.uint8), pinned((m, h, w), np.uint8)
        arms = {
            "float2": lambda: e.calc_batch(list(fr), 1, flows=flows),
            "planes": lambda: e.calc_batch_planes(list(fr), 1, out=planes),
            "u8": lambda: e.calc_batch_u8_into(list(fr), 1, 20, qx, qy),
        }
        for f in arms.values():
            f()
        best = {k: 0.0 for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                t = time.perf_counter()
                f()
                best[k] = max(best[k], m / (time.perf_counter() - t))
        assert planes.tobytes() == np.ascontiguousarray(np.moveaxis(flows, -1, 1)).tobytes()
        res["calls"]["%dx%d" % (w, h)] = {k + "_pairs_per_s": round(v, 2) for k, v in best.items()}
        if w == 1920:
            planes_1080 = planes.copy()
        e.release()
    shm = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    disk = a.disk or tempfile.mkdtemp()
    res["writer_MBps"]["tmpfs"] = round(write_rate(planes_1080, shm, a.rounds), 1)
    res["writer_MBps"]["disk"] = round(write_rate(planes_1080, disk, a.rounds), 1)
    res["disk_dir_fs"] = subprocess.run(["stat", "-f", "-c", "%T", disk], capture_output=True, text=True).stdout.strip()
    if not a.disk:
        os.rmdir(disk)
    pair_mb = 1920 * 1080 * 8 / 1e6
    calls = res["calls"]["1920x1080"]
    res["bound_1080p"] = {
        "planes_call_MBps": round(calls["planes_pairs_per_s"] * pair_mb, 1),
        "file_write_bounds_tmpfs": res["writer_MBps"]["tmpfs"] < calls["planes_pairs_per_s"] * pair_mb,
        "file_write_bounds_disk": res["writer_MBps"]["disk"] < calls["planes_pairs_per_s"] * pair_mb,
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
