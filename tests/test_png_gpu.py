"""GPU convertFlowToPngImage (SURVEY §8 f4, /root/reference/src/common.cpp:18-46) bit-exact against the numpy restatement
(oracle/cv_restate.py, itself pinned to cv2 in tests/test_preproc_cpu.py)."""
import numpy as np
import pytest

from denseflow_b200 import synth
from oracle import cv_restate as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", [(64, 96, 0.7), (255, 341, 6.0), (120, 33, 20.0), (77, 201, 2.5), (1080, 1920, 3.0), (40, 50, 900.0)])
def test_png_image_is_bit_exact(case):
    import torch
    import denseflow_b200 as d
    h, w, scale = case
    rng = np.random.default_rng(h * 1000 + w)
    flow = (rng.standard_normal((h, w, 2)) * scale).astype(np.float32)
    if scale > 100:
        flow[3, 4] = (5000.0, -4000.0)  # larger than the frame: clipped to the extent
    e = d.create("tvl1", 0, 64, 64)
    for _ in range(2):  # twice: the reduction's ticket must re-arm itself
        bgr, bounds = e.flow_to_png_image_device(torch.from_numpy(flow).cuda())
        torch.cuda.synchronize()
        want, bx, by = R.flow_to_png_image(flow)
        assert bounds == (bx, by)
        assert np.array_equal(bgr.cpu().numpy(), want)


def test_png_image_of_an_engine_flow():
    import torch
    import denseflow_b200 as d
    a, b, _ = synth.pair(96, 128, 4)
    e = d.create("farn", 0, 128, 96)
    flow = e.calc(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    bgr, bounds = e.flow_to_png_image_device(flow)
    torch.cuda.synchronize()
    want, bx, by = R.flow_to_png_image(flow.cpu().numpy())
    assert bounds == (bx, by) and np.array_equal(bgr.cpu().numpy(), want)
    import cv2
    ok, png = cv2.imencode(".png", bgr.cpu().numpy())  # encodeFlowMapPng's last step stays on the host (lossless)
    assert ok and np.array_equal(cv2.imdecode(png, cv2.IMREAD_COLOR), want)


def _png_check(e, flow, pitch_extra=0):
    import torch
    h, w = flow.shape[:2]
    dev = torch.full((h, w + pitch_extra, 2), float("nan"), dtype=torch.float32, device="cuda")[:, :w]
    dev.copy_(torch.from_numpy(flow))
    bgr, bounds = e.flow_to_png_image_device(dev)
    torch.cuda.synchronize()
    want, bx, by = R.flow_to_png_image(flow)
    assert bounds == (bx, by), ((h, w), bounds, (bx, by))
    assert np.array_equal(bgr.cpu().numpy(), want), (h, w)
    return bx, by


# (h, w): h = 1, 2, 3 (half_h and split degenerate) and w = 1; fewer than 256 pixels (one partial block); kPngPackBlocks x 256
# = 135168 pixels +- 1 (kPngPackBlocks = 528): the min/max grid stops growing there and the grid-stride loop takes over
PNG_SHAPES = [(1, 1), (1, 7), (2, 1), (2, 5), (3, 1), (3, 9), (7, 1), (1100, 1), (1, 1100), (15, 17), (1, 255), (1, 256), (1, 257),
              (1, 135167), (256, 528), (3, 45056), (1, 135169), (367, 369)]


@pytest.mark.parametrize("pitch_extra", [0, 3])
@pytest.mark.parametrize("shape", PNG_SHAPES)
def test_png_image_at_degenerate_sizes(shape, pitch_extra):
    import denseflow_b200 as d
    h, w = shape
    e = d.create("tvl1", 0, 64, 64)
    rng = np.random.default_rng(h * 7 + w)
    flow = (rng.standard_normal((h, w, 2)) * 3).astype(np.float32)
    _png_check(e, flow, pitch_extra)
    if h * w > 1:  # the extremes in the last pixel (the grid-stride loop's tail), then in the first
        flow[-1, -1] = (-40.0, 41.0)
        _png_check(e, flow, pitch_extra)
        flow[0, 0] = (55.0, -56.0)
        _png_check(e, flow, pitch_extra)


def test_png_bounds_on_the_multiple_of_8_rule_and_the_cap():
    """max |flow| placed where ceil(m * 128 / 127 / 4) * 4 is a multiple of 8 (the bound then gets + 4), one float either side
    of it, and past 255 * 4 (the cap, reached only when the frame extent allows it)"""
    import denseflow_b200 as d
    e = d.create("tvl1", 0, 64, 64)
    for h, w in [(1100, 2), (2, 1100), (3, 1), (1, 3)]:
        for k in (1, 2, 3, 63, 126, 127):
            m = np.float32(8 * k * 127 / 128)
            for v in (np.nextafter(m, np.float32(0)), m, np.nextafter(m, np.float32(np.inf))):
                flow = np.zeros((h, w, 2), np.float32)
                flow[h // 2, w // 2] = (v, -v)
                bx, by = _png_check(e, flow)
                assert bx % 8 == 4 and by % 8 == 4
        flow = np.zeros((h, w, 2), np.float32)
        flow[0, -1] = (5000.0, -5000.0)
        bx, by = _png_check(e, flow)
        assert (bx == 1020) == (w >= 1013) and (by == 1020) == (h >= 1013)
