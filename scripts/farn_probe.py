"""Farneback throughput (device-resident frames, 16 pairs per call) and iteration-kernel bandwidth per build variant."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import denseflow_b200 as d
from denseflow_b200 import synth
variants = sys.argv[1].split(",") if len(sys.argv) > 1 else ["default"]
sizes = [(1280, 720), (1920, 1080), (340, 256)] if len(sys.argv) < 3 else [tuple(int(v) for v in s.split("x")) for s in sys.argv[2].split(",")]
for (W, H) in sizes:
    N = 17
    fr = synth.stream(H, W, N, seed=2)
    dev = torch.from_numpy(fr).cuda()
    out = torch.empty((N - 1, H, W, 2), dtype=torch.float32, device="cuda")
    for variant in variants:
        e = d.FarnebackOpticalFlow.create(0, W, H, variant)
        e.set("time_kernels", 1)
        for _ in range(2):
            e.calc_batch_device(dev, 1, out)
        torch.cuda.synchronize(); e.reset_counters()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(3):
            e.calc_batch_device(dev, 1, out)
        ev1.record(); torch.cuda.synchronize()
        dt = ev0.elapsed_time(ev1) / 1e3 / 3
        c = e.counters()
        kt = max(c["timed_kernel_ns"], 1) / 1e9 / 3
        print("%s " % variant, end="")
        print("%dx%d: %.3f ms/pair (%.1f pairs/s); iteration kernels %.3f ms/pair = %.0f GB/s at 88 B/px.iter" % (
            W, H, dt / (N - 1) * 1e3, (N - 1) / dt, kt / (N - 1) * 1e3, 88.0 * c["pixel_iters"] / 3 / kt / 1e9))
        e.release()
