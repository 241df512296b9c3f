"""dfb_calc_device on two frames whose rows lie at different pitches: each frame is prepared with its own pitch, the flow is
byte-identical to calc_batch on the same frames (the batched frame preparation of the host calls), and one call launches
a fixed number of kernels, for both engines in both builds."""
import numpy as np
import pytest

from denseflow_b200 import synth

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
SIZES = [(64, 64), (341, 257), (1001, 37)]  # (w, h); 1001 x 37: an odd width, four TV-L1 levels and one Farneback level

# kernel launches of one call at the create() defaults.  TV-L1 (5, 5 and 4 levels): per frame one u8-to-float launch and
# nscales - 1 resizes, then the fused pair kernel.  Farneback (2, 4 and 1 levels): per frame one u8-to-float launch, then per
# level the level image (one launch at full resolution, two below) and the polynomial expansion; per level of the pair the
# flow start, the matrices and 10 iterations, and the merge.
LAUNCHES = {
    ("tvl1", 64, 64): 2 * 5 + 1,
    ("tvl1", 341, 257): 2 * 5 + 1,
    ("tvl1", 1001, 37): 2 * 4 + 1,
    ("farn", 64, 64): 2 * (1 + 3 + 2) + 2 * 12 + 1,
    ("farn", 341, 257): 2 * (1 + 3 * 3 + 2) + 4 * 12 + 1,
    ("farn", 1001, 37): 2 * (1 + 2) + 12 + 1,
}


def _pitched(frame, pitch):
    """a CUDA view of `frame` whose rows are `pitch` bytes apart"""
    import torch
    h, w = frame.shape
    buf = torch.zeros((h, pitch), dtype=torch.uint8, device="cuda")
    view = buf[:, :w]
    view.copy_(torch.from_numpy(frame))
    assert view.stride(0) == pitch
    return view


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_calc_device_at_two_pitches(alg, variant):
    import torch
    import denseflow_b200 as d
    e = d.create(alg, 0, 1024, 512, variant)
    for k, (w, h) in enumerate(SIZES):
        a, b, _ = synth.pair(h, w, k)
        want = e.calc_batch([a, b])[0]
        base = (w + 3) & ~3
        va, vb = _pitched(a, base + 1), _pitched(b, base + 64)  # a's pitch is not a multiple of 4
        torch.cuda.synchronize()
        before = e.counters()["kernel_launches"]
        flow = e.calc(va, vb)
        torch.cuda.synchronize()
        launches = e.counters()["kernel_launches"] - before
        got = flow.cpu().numpy()
        bad = got.view(np.int32) != want.view(np.int32)
        assert not bad.any(), "%dx%d: %d of %d differ from calc_batch" % (w, h, bad.sum(), bad.size)
        assert launches == LAUNCHES[(alg, w, h)], (w, h, launches)
    e.release()
