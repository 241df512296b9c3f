"""1080p throughput of the fused engine vs lanes / k (device-resident frames, 16 pairs per call)."""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import denseflow_b200 as d
from denseflow_b200 import synth

W, H = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (1920, 1080)
N = int(sys.argv[4]) if len(sys.argv) > 4 else 17
fr = synth.stream(H, W, N, seed=1)
dev = torch.from_numpy(fr).cuda()
out = torch.empty((N - 1, H, W, 2), dtype=torch.float32, device="cuda")
ref = None
variants = sys.argv[3].split(',') if len(sys.argv) > 3 else ['default']
ks = [int(x) for x in sys.argv[5].split(',')] if len(sys.argv) > 5 else [8]
lane_list = [int(x) for x in sys.argv[6].split(',')] if len(sys.argv) > 6 else [1, 0]
cfgs = [(v, l, k, 1) for v in variants for k in ks for l in lane_list]
for variant, lanes, k, fs in cfgs:
    e = d.OpticalFlowDual_TVL1.create(0, W, H, variant)
    e.set("lanes", lanes); e.set("fused_k", k)
    e.calc_batch_device(dev, 1, out); torch.cuda.synchronize()
    e.reset_counters()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(); e.calc_batch_device(dev, 1, out); ev1.record(); torch.cuda.synchronize()
    dt = ev0.elapsed_time(ev1) / 1e3
    c = e.counters()
    res = out.cpu().numpy()
    if ref is None: ref = res.copy()
    print("%s " % variant, end=""); print("lanes=%d k=%d: %.3f ms/pair (%.1f pairs/s), launches %d, px-iters/pair %.1fM, max|diff| vs lanes=1: %.2e" % (
        lanes, k, dt / (N - 1) * 1e3, (N - 1) / dt, c["kernel_launches"], c["pixel_iters"] / (N - 1) / 1e6, np.abs(res - ref).max()))
    e.release()
