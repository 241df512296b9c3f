"""`python -m denseflow_b200` with a video's windows shared among the workers (`ListRunner.run_windows`, what the command
runs) against whole videos per worker (`ListRunner.run_stream`, what it ran before), on single long inputs and on a list.

Workloads, written to a temporary directory (the list with scripts/cli_bench.py's writer; the long inputs 50 frames at a
time, so a 600-frame 1080p stream never sits in memory whole):
  - one 1920x1080 `-if` folder of 600 q95 frames, TV-L1;
  - one 1920x1080 FFV1 video of 300 frames, TV-L1;
  - one 340x256 FFV1 video of 2000 frames, Farneback;
  - the 340x256 FFV1 list of DESIGN §7: 6 videos of 100 frames, TV-L1.
Each runs `-s=1 -b=20 -st=jpg` through the command's own readers and file writes, in a fresh process, two workers on every
visible GPU.  The arms alternate, 3 rounds each after one warm-up of each, and flows/s come from the command's summary line.
With more than one GPU visible, the 1/2/4/8-GPU subsets run too, each with CUDA_VISIBLE_DEVICES set.  Prints the GPU name
and power limit and one JSON line.

    python scripts/window_bench.py [--rounds 3] [--only NAME] [--out FILE]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from cli_bench import SUMMARY, card, write_inputs  # noqa: E402
from denseflow_b200 import synth  # noqa: E402

# the command in a child process; arm "stream" puts run_stream where the command calls run_windows
CHILD = """
import sys
from denseflow_b200 import cli, listrun
if sys.argv[1] == "stream":
    listrun.ListRunner.run_windows = listrun.ListRunner.run_stream
sys.exit(cli.main(sys.argv[2:]))
"""


def frames(n, h, w, seed):
    """n BGR frames of one synthetic stream, made 50 at a time."""
    for t0 in range(0, n, 50):
        for g in synth.stream(h, w, min(50, n - t0), seed=seed, phase=t0):
            yield np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8)


def write_video(path, n, h, w, seed):
    import cv2
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"FFV1"), 25, (w, h))
    for f in frames(n, h, w, seed):
        vw.write(f)
    vw.release()
    return path


def write_folder(path, n, h, w, seed):
    import cv2
    os.makedirs(path, exist_ok=True)
    for i, f in enumerate(frames(n, h, w, seed)):
        with open(os.path.join(path, "img_%05d.jpg" % i), "wb") as fh:
            fh.write(cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes())
    return path


def run_cli(arm, args, out_dir, env):
    shutil.rmtree(out_dir, ignore_errors=True)
    r = subprocess.run([sys.executable, "-c", CHILD, arm] + args + ["-s=1", "-b=20", "-st=jpg", "-o=" + out_dir], cwd=ROOT,
                       capture_output=True, text=True, env=env)
    m = SUMMARY.search(r.stdout)
    if r.returncode != 0 or not m:
        raise RuntimeError("command failed (%d): %s %s" % (r.returncode, r.stdout[-2000:], r.stderr[-2000:]))
    return float(m.group(6))


def measure(args, tmp, rounds, env):
    out_dir = os.path.join(tmp, "out")
    for arm in ("stream", "windows"):
        run_cli(arm, args, out_dir, env)  # warm-up: imports, contexts, page cache
    got = {"stream": [], "windows": []}
    for _ in range(rounds):
        for arm in ("stream", "windows"):
            got[arm].append(round(run_cli(arm, args, out_dir, env), 1))
    return {"stream_flows_per_s": got["stream"], "windows_flows_per_s": got["windows"],
            "windows_over_stream": round(float(np.median(got["windows"]) / np.median(got["stream"])), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default=None, help="run only the workloads whose name contains this")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    name, power = card()
    ngpu = torch.cuda.device_count()
    res = {"card": name, "power_limit": power, "gpus": ngpu, "workers_per_gpu": 2, "host_cores": len(os.sched_getaffinity(0)),
           "results": {}}
    print("card: %s, power limit %s, %d GPU(s)" % (name, power, ngpu), flush=True)
    tmp = tempfile.mkdtemp(prefix="dfb_window_bench_")
    try:
        writers = [
            ("1920x1080_if_600_tvl1", lambda: [write_folder(os.path.join(tmp, "if1080"), 600, 1080, 1920, 310), "-if", "-a=tvl1"]),
            ("1920x1080_ffv1_300_tvl1", lambda: [write_video(os.path.join(tmp, "v1080.avi"), 300, 1080, 1920, 311), "-a=tvl1"]),
            ("340x256_ffv1_2000_farn", lambda: [write_video(os.path.join(tmp, "v256.avi"), 2000, 256, 340, 312), "-a=farn"]),
            ("340x256_ffv1_list_6x100_tvl1", lambda: [write_inputs(tmp, "340x256", 6, 100, 256, 340)["ffv1"], "-a=tvl1"]),
        ]
        workloads = [(key, write()) for key, write in writers if a.only is None or a.only in key]
        subsets = [g for g in (1, 2, 4, 8) if g < ngpu] + [ngpu]
        for g in subsets:
            env = dict(os.environ, PYTHONPATH=ROOT)
            if g != ngpu:
                env["CUDA_VISIBLE_DEVICES"] = ",".join(str(d) for d in range(g))
            for key, args in workloads:
                r = measure(args, tmp, a.rounds, env)
                res["results"]["%s_%dgpu" % (key, g)] = r
                print("%s, %d GPU(s): %s" % (key, g, r), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
