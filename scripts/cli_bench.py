"""`python -m denseflow_b200` on generated video lists: frames/s and flows/s from the command's own summary line, next to
`ListRunner.run_videos` on the same frames already decoded, so the cost of decoding on the host shows.

Inputs, written to a temporary directory with cv2.VideoWriter: FFV1 (lossless) and MJPG `.avi` files and `-if` folders of
q95 JPEG frames, as 340x256 clips and 1920x1080 streams.  Each list runs `-a=tvl1|farn -s=1 -b=20 -st=jpg` once as a warm-up
and then timed; every visible GPU runs two workers, in both arms.  Prints the GPU name and power limit and one JSON line.

    python scripts/cli_bench.py [--clips 8] [--clip-frames 120] [--streams 2] [--stream-frames 120] [--out FILE]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from denseflow_b200 import cli, listrun, synth  # noqa: E402

SUMMARY = re.compile(r"(\d+) videos \((\d+) frames, (\d+) \w+ flows\) processed, using ([^s]+)s, decoding speed (\S+)fps, "
                     r"flow speed (\S+)fps")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def frames(n, h, w, seed):
    gray = synth.stream(h, w, n, seed=seed)
    return [np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8) for g in gray]


def write_inputs(root, name, n_videos, n_frames, h, w):
    """Per format, a list.txt of n_videos inputs: FFV1 and MJPG videos, and `-if` folders."""
    import cv2
    lists = {fmt: [] for fmt in ("ffv1", "mjpg", "if")}
    for v in range(n_videos):
        fr = frames(n_frames, h, w, seed=200 + v)
        for fmt, fourcc in (("ffv1", "FFV1"), ("mjpg", "MJPG")):
            p = os.path.join(root, "%s_%s" % (name, fmt), "v%02d.avi" % v)
            os.makedirs(os.path.dirname(p), exist_ok=True)
            vw = cv2.VideoWriter(p, cv2.VideoWriter_fourcc(*fourcc), 25, (w, h))
            for f in fr:
                vw.write(f)
            vw.release()
            lists[fmt].append(p)
        d = os.path.join(root, "%s_if" % name, "v%02d" % v)
        os.makedirs(d, exist_ok=True)
        for i, f in enumerate(fr):
            with open(os.path.join(d, "img_%05d.jpg" % i), "wb") as fh:
                fh.write(cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes())
        lists["if"].append(d)
    out = {}
    for fmt, paths in lists.items():
        out[fmt] = os.path.join(root, "%s_%s.txt" % (name, fmt))
        with open(out[fmt], "w") as fh:
            fh.write("".join(p + "\n" for p in paths))
    return out


def run_cli(lst, alg, use_frames, out_dir):
    shutil.rmtree(out_dir, ignore_errors=True)
    args = [sys.executable, "-m", "denseflow_b200", lst, "-a=" + alg, "-s=1", "-b=20", "-o=" + out_dir] + (["-if"] if use_frames else [])
    r = subprocess.run(args, cwd=ROOT, capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT))
    m = SUMMARY.search(r.stdout)
    if r.returncode != 0 or not m:
        raise RuntimeError("command failed (%d): %s %s" % (r.returncode, r.stdout[-2000:], r.stderr[-2000:]))
    return {"frames": int(m.group(2)), "flows": int(m.group(3)), "seconds": float(m.group(4)), "frames_per_s": float(m.group(5)),
            "flows_per_s": float(m.group(6))}


def decoded(lst, use_frames):
    """What the command's source hands the runner, decoded up front: BGR frames, or the JPEG files' bytes."""
    import cv2
    videos = []
    for p in cli.read_list(lst):
        if use_frames:
            videos.append([open(f, "rb").read() for f in cli.frame_files(p)])
            continue
        cap, fr = cv2.VideoCapture(p), []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            fr.append(f)
        videos.append(fr)
    return videos


def run_videos(alg, devices, videos, w, h):
    r = listrun.ListRunner(alg, devices, w, h)
    try:
        r.run_videos(videos[:1], step=1, bound=20, jpeg_exact=1, chunk_flows=cli.CHUNK_FLOWS, on_chunk=lambda *a: None)  # warm-up
        t0 = time.perf_counter()
        st = r.run_videos(videos, step=1, bound=20, jpeg_exact=1, chunk_flows=cli.CHUNK_FLOWS, on_chunk=lambda *a: None)
        sec = time.perf_counter() - t0
    finally:
        r.close()
    return {"frames": st["frames"], "flows": st["flows"], "seconds": round(sec, 3), "frames_per_s": round(st["frames"] / sec, 1),
            "flows_per_s": round(st["flows"] / sec, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=8)
    ap.add_argument("--clip-frames", type=int, default=120)
    ap.add_argument("--streams", type=int, default=2)
    ap.add_argument("--stream-frames", type=int, default=120)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    name, power = card()
    ngpu = torch.cuda.device_count()
    devices = [d for d in range(ngpu) for _ in range(cli.WORKERS_PER_DEVICE)]
    res = {"card": name, "power_limit": power, "gpus": ngpu, "host_cores": len(os.sched_getaffinity(0)), "results": {}}
    print("card: %s, power limit %s, %d GPU(s)" % (name, power, ngpu), flush=True)
    tmp = tempfile.mkdtemp(prefix="dfb_cli_bench_")
    try:
        for size, n_videos, n_frames, h, w in (("340x256", a.clips, a.clip_frames, 256, 340),
                                               ("1920x1080", a.streams, a.stream_frames, 1080, 1920)):
            lists = write_inputs(tmp, size, n_videos, n_frames, h, w)
            for fmt, lst in lists.items():
                use_frames = fmt == "if"
                videos = decoded(lst, use_frames)
                for alg in ("tvl1", "farn"):
                    out_dir = os.path.join(tmp, "out")
                    run_cli(lst, alg, use_frames, out_dir)  # warm-up: imports, contexts, handles
                    got = run_cli(lst, alg, use_frames, out_dir)
                    ref = run_videos(alg, devices, videos, w, h)
                    key = "%s_%s_%s" % (size, fmt, alg)
                    res["results"][key] = {"videos": n_videos, "frames_per_video": n_frames, "cli": got, "run_videos_decoded": ref,
                                           "cli_over_run_videos": round(got["flows_per_s"] / ref["flows_per_s"], 3)}
                    print(key, res["results"][key], flush=True)
                del videos
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
