"""TV-L1 (or Farneback) on video with and without `use_initial_flow`: a cold start for every pair against a warm start where
pair i of a stream starts from pair i - 1's flow.

Workloads: K independent `synth.stream` clips, each of N frames, at 1920x1080 and at 340x256, resident in HBM.  One
`calc_batch_device` call solves pair i of all K streams side by side (frames ordered stream-major per time step, step K),
so the lanes stay busy as they do on a list of videos.  Both arms pass the same device flow buffer; the warm arm reads it
as the start, so pair i starts from pair i - 1's flow (zeros for the first pair, which gives the cold start's bits), and
the cold arm ignores it.  The arms alternate, `--rounds` times each after one warm-up round; pairs/s is the best round's.
Reported per arm:
  - pairs/s (host clock around each call and a device synchronise, pairs after the first of each stream);
  - mean executed inner iterations per (scale, warp) of the pairs after the first, from dfb_get_tvl1_pair_stats (TV-L1 only);
  - AEE against the synthetic ground truth, and warm against cold.
The ground truth is first order: frame t is the texture displaced by (X_t, Y_t) (synth.stream), so the flow from t to
t + 1 is taken as (X_{t+1} - X_t, Y_{t+1} - Y_t) at each pixel.  Prints the GPU name and power limit and one JSON line.

    python scripts/warm_start_bench.py [--alg tvl1|farn] [--rounds 3] [--frames 11] [--only 1080p|340x256] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from cli_bench import card  # noqa: E402
from denseflow_b200 import synth  # noqa: E402

# (name, width, height, streams per call): 7 pairs fill the 1080p lanes, 64 the 340x256 ones (the calc calls' group size)
WORKLOADS = [("1080p", 1920, 1080, 7), ("340x256", 340, 256, 64)]


def ground_truth(h, w, t):
    """synth.stream's displacement from frame t to t + 1, first order"""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)

    def disp(tt):
        X = 12 * np.sin(2 * np.pi * tt / 50) + 1.5 * np.sin(2 * np.pi * yy / h + tt / 20)
        Y = 8 * np.cos(2 * np.pi * tt / 70) + 1.0 * np.cos(2 * np.pi * xx / w + tt / 25)
        return X, Y

    X0, Y0 = disp(t)
    X1, Y1 = disp(t + 1)
    return np.stack([X1 - X0, Y1 - Y0], -1).astype(np.float32)


def aee(f, g):
    """mean end-point error of two [T, K, H, W, 2] stacks, one time step at a time"""
    return float(np.mean([synth.aee(f[i], g[i]) for i in range(len(f))]))


def run_arm(e, clips, warm, alg):
    """every pair of every clip, device-resident (frames and flows in HBM, `calc_batch_device`), so the numbers are the GPU's
    and not the host copies'; returns (flows [T-1, K, H, W, 2] on the host, seconds after the first pair, iterations per
    (scale, warp))"""
    import torch
    K, T, h, w = clips.shape
    e.set("use_initial_flow", 1 if warm else 0)
    flows = np.zeros((T - 1, K, h, w, 2), np.float32)
    dflow = torch.zeros((K, h, w, 2), dtype=torch.float32, device="cuda")  # the warm arm's chain: pair i reads pair i - 1's
    iters = []
    secs = 0.0
    for i in range(T - 1):
        frames = torch.cat([clips[:, i], clips[:, i + 1]])  # [2K, H, W]: pair k = (k, k + K)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e.calc_batch_device(frames, step=K, flows=dflow)
        torch.cuda.synchronize()
        if i > 0:
            secs += time.perf_counter() - t0
        flows[i] = dflow.cpu().numpy()
        if alg == "tvl1" and i > 0:
            for k in range(K):
                log = e.tvl1_pair_stats(k)
                iters.append(log[log.sum(1) > 0])
    it = float(np.mean(np.concatenate([x.ravel() for x in iters]))) if iters else None
    return flows, secs, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--alg", default="tvl1", choices=["tvl1", "farn"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=11)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import denseflow_b200 as d
    name, power = card()
    print("GPU: %s, power limit %s" % (name, power))
    result = {"gpu": name, "power_limit": power, "alg": args.alg, "frames_per_stream": args.frames, "workloads": {}}
    for wl, w, h, K in WORKLOADS:
        if args.only and wl != args.only:
            continue
        import torch
        clips = torch.from_numpy(np.stack([synth.stream(h, w, args.frames, seed=100 + k) for k in range(K)])).cuda()
        gt = np.stack([ground_truth(h, w, t) for t in range(args.frames - 1)])  # every clip moves alike; textures differ
        e = d.create(args.alg, 0, w, h)
        best = {"cold": None, "warm": None}
        res = {}
        for r in range(args.rounds + 1):
            for arm in ("cold", "warm"):
                flows, secs, it = run_arm(e, clips, arm == "warm", args.alg)
                if r == 0:
                    res[arm] = (flows, it)
                    continue
                rate = (args.frames - 2) * K / secs
                best[arm] = rate if best[arm] is None else max(best[arm], rate)
        (fc, ic), (fw, iw) = res["cold"], res["warm"]
        gtb = np.broadcast_to(gt[:, None], fc.shape)
        row = {"width": w, "height": h, "streams_per_call": K,
               "cold": {"pairs_per_s": best["cold"], "mean_iters_per_scale_warp": ic, "aee_vs_truth_px": aee(fc, gtb)},
               "warm": {"pairs_per_s": best["warm"], "mean_iters_per_scale_warp": iw, "aee_vs_truth_px": aee(fw, gtb)},
               "aee_warm_vs_cold_px": aee(fw, fc),
               "first_pair_bits_equal": bool(np.array_equal(fw[0], fc[0]))}
        result["workloads"][wl] = row
        print("%s %s: cold %.1f pairs/s, %s iters/(scale, warp), AEE vs truth %.4f px | warm %.1f pairs/s, %s iters, AEE %.4f px | "
              "warm vs cold %.4f px" % (args.alg, wl, best["cold"], ic, row["cold"]["aee_vs_truth_px"], best["warm"], iw,
                                        row["warm"]["aee_vs_truth_px"], row["aee_warm_vs_cold_px"]), flush=True)
        e.release()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
