"""GPU BGR->gray and INTER_LINEAR uint8 resize (SURVEY §8 f3) — bit-exact vs the OpenCV restatements."""
import numpy as np
import pytest

import geometry_cases as gc
from oracle import cv_restate as R

pytestmark = pytest.mark.gpu


def _engine():
    import denseflow_b200 as d
    return d.OpticalFlowDual_TVL1.create(0, 64, 64)


def test_bgr_to_gray_bit_exact():
    import torch
    rng = np.random.default_rng(0)
    e = _engine()
    for shape in [(97, 131), (1080, 1920), (1, 1)]:
        bgr = rng.integers(0, 256, shape + (3,), dtype=np.uint8)
        g = e.bgr_to_gray_device(torch.from_numpy(bgr).cuda()).cpu().numpy()
        assert np.array_equal(g, R.bgr2gray(bgr))


@pytest.mark.parametrize("case", [((240, 320), (160, 120)), ((240, 320), (341, 256)), ((240, 320), (400, 300)), ((1080, 1920), (455, 256)),
                                  ((480, 640), (340, 256)), ((77, 100), (33, 500)), ((240, 320), (320, 240))])
def test_resize_bit_exact(case):
    import torch
    (sh, sw), (dw, dh) = case
    rng = np.random.default_rng(2)
    src = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
    e = _engine()
    out = e.resize_gray_device(torch.from_numpy(src).cuda(), dw, dh).cpu().numpy()
    assert np.array_equal(out, R.resize_linear_u8(src, dw, dh))


def _offset_view(img, off, extra):
    """img (uint8, [h, w] or [h, w, 3]) copied into a device buffer whose rows are `extra` bytes longer than the image and
    whose base is `off` bytes past an aligned address"""
    import torch
    h, row = img.shape[0], img[0].size
    pitch = row + extra
    buf = torch.zeros(h * pitch + off, dtype=torch.uint8, device="cuda")
    shape, stride = (img.shape, (pitch, 3, 1)) if img.ndim == 3 else (img.shape, (pitch, 1))
    v = torch.as_strided(buf, shape, stride, off)
    v.copy_(torch.from_numpy(img))
    assert v.data_ptr() % 4 == off % 4 and v.stride(0) == pitch
    return v


@pytest.mark.parametrize("off, extra", [(1, 3), (2, 5), (3, 64)])
def test_bgr_to_gray_from_pitched_offset_buffers(off, extra):
    import torch
    rng = np.random.default_rng(off)
    e = _engine()
    for w, h in gc.TINY[::5] + [(1, 1920), (1920, 1), (7, 1080), (1080, 7), (131, 97)]:
        bgr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        g = e.bgr_to_gray_device(_offset_view(bgr, off, extra))
        torch.cuda.synchronize()
        assert np.array_equal(g.cpu().numpy(), R.bgr2gray(bgr)), (w, h)


@pytest.mark.parametrize("off, extra", [(0, 0), (1, 3), (3, 17)])
@pytest.mark.parametrize("src, dst", gc.RESIZE_CASES)
def test_resize_at_degenerate_sizes_from_pitched_offset_buffers(src, dst, off, extra):
    import torch
    (sw, sh), (dw, dh) = src, dst
    img = np.random.default_rng(sw * 7 + sh).integers(0, 256, (sh, sw), dtype=np.uint8)
    out = _engine().resize_gray_device(_offset_view(img, off, extra), dw, dh)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), R.resize_linear_u8(img, dw, dh))
