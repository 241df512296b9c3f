"""The gray / resize restatements (oracle/cv_restate.py) against real OpenCV CPU code (cv2 is in the image)."""
import numpy as np
import pytest

import geometry_cases as gc
from oracle import cv_restate as R

cv2 = pytest.importorskip("cv2")


def test_bgr2gray_matches_opencv():
    rng = np.random.default_rng(0)
    bgr = rng.integers(0, 256, (97, 131, 3), dtype=np.uint8)
    assert np.array_equal(R.bgr2gray(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))
    ramp = np.stack(np.meshgrid(np.arange(256), np.arange(256)), -1).astype(np.uint8)
    full = np.concatenate([ramp, np.full((256, 256, 1), 77, np.uint8)], -1)
    assert np.array_equal(R.bgr2gray(full), cv2.cvtColor(full, cv2.COLOR_BGR2GRAY))


def test_bgr2gray_matches_opencv_on_every_triple():
    """all 2^24 BGR triples, as 16 images of 1024 x 1024"""
    for chunk in range(16):
        i = np.arange(chunk << 20, (chunk + 1) << 20, dtype=np.uint32)
        bgr = np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(1024, 1024, 3)
        assert np.array_equal(R.bgr2gray(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)), chunk


@pytest.mark.parametrize("dst", [(160, 120), (341, 256), (224, 224), (400, 300), (455, 256), (256, 341), (100, 77), (639, 479),
                                 (340, 256), (33, 500), (320, 240)])
def test_resize_linear_u8_matches_opencv(dst):
    rng = np.random.default_rng(1)
    src = rng.integers(0, 256, (240, 320), dtype=np.uint8)
    dw, dh = dst
    assert np.array_equal(R.resize_linear_u8(src, dw, dh), cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR))


@pytest.mark.parametrize("src, dst", gc.RESIZE_CASES)
def test_resize_linear_u8_matches_opencv_at_degenerate_sizes(src, dst):
    (sw, sh), (dw, dh) = src, dst
    img = np.random.default_rng(sw * 7 + sh).integers(0, 256, (sh, sw), dtype=np.uint8)
    assert np.array_equal(R.resize_linear_u8(img, dw, dh), cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR))


def test_new_size_rules():
    # DenseFlow::get_new_size, /root/reference/src/denseflow_gpu.cpp:57-78
    assert R.new_size(1920, 1080, new_short=256) == (True, 455, 256)
    assert R.new_size(320, 240, new_short=256) == (False, 320, 240)  # ns only shrinks
    assert R.new_size(1080, 1920, new_short=256) == (True, 256, 455)
    assert R.new_size(640, 480, new_width=340) == (True, 340, 255)
    assert R.new_size(640, 480, new_height=256) == (True, 341, 256)
    assert R.new_size(640, 480, 340, 256) == (True, 340, 256)


def test_flow_to_png_image_pieces_match_opencv():
    """convertFlowToPngImage (/root/reference/src/common.cpp:18-46) piece by piece against the cv2 calls it makes."""
    rng = np.random.default_rng(3)
    for (h, w, scale) in [(64, 96, 0.7), (255, 341, 6.0), (120, 33, 20.0), (77, 201, 2.5)]:
        flow = (rng.standard_normal((h, w, 2)) * scale).astype(np.float32)
        img, bx, by = R.flow_to_png_image(flow)
        fx, fy = np.ascontiguousarray(flow[..., 0]), np.ascontiguousarray(flow[..., 1])
        for comp, ext, b in ((fx, w, bx), (fy, h, by)):
            mn, mx, _, _ = cv2.minMaxLoc(comp)
            want = min(255. * 4, np.ceil((min(float(ext), max(abs(mn), abs(mx))) * 128. / 127.) / 4) * 4)
            if int(want) % 8 == 0:
                want += 4
            assert b == want and b % 4 == 0 and int(b) % 8 != 0
        # Mat::convertTo(CV_8U, alpha, 128): cv2 exposes the same cvtScale kernel as convertScaleAbs (|.| of a non-negative value)
        for c, comp, b in ((0, fx, bx), (1, fy, by)):
            alpha = float(np.float32(1. / ((1. / 128.) * b)))
            if (comp.astype(np.float64) * alpha + 128 >= 0.5).all():
                assert np.array_equal(img[..., c], cv2.convertScaleAbs(comp, alpha=alpha, beta=128.0))
        # third channel: two FILLED rectangles with cv::Point's double -> int truncation
        bch = np.zeros((h, w), np.uint8)
        cv2.rectangle(bch, (0, 0), (w - 1, int(h / 2)), int(bx / 4), cv2.FILLED)
        cv2.rectangle(bch, (0, int(h / 2 + 1)), (w - 1, h - 1), int(by / 4), cv2.FILLED)
        assert np.array_equal(img[..., 2], bch)
    # a flow larger than the frame is clipped to the extent, and the bound saturates at 255 * 4
    big = np.zeros((40, 50, 2), np.float32)
    big[0, 0] = (5000.0, -3.0)
    _, bx, by = R.flow_to_png_image(big)
    assert bx == np.ceil(50 * 128. / 127. / 4) * 4 and by == 4.0
