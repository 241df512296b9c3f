"""Numpy restatement of what the frame-extraction mode (`-s=0`) computes before the JPEG DCT: cv::resize(INTER_LINEAR) of
the colour frame, then libjpeg's JFIF colour conversion and 4:2:0 chroma downsampling.  Test infrastructure, pinned live
against cv2 and libjpeg-turbo (through Pillow) in tests/test_extract_cpu.py; the CUDA kernel is checked against it."""
import numpy as np

from oracle import cv_restate as R


def resize_linear_u8c(src, dw, dh):
    """cv::resize(src, (dw, dh), INTER_LINEAR) for CV_8UC1 or CV_8UC3: the CV_8UC1 arithmetic on every channel."""
    if src.ndim == 2:
        return R.resize_linear_u8(src, dw, dh)
    return np.stack([R.resize_linear_u8(np.ascontiguousarray(src[..., c]), dw, dh) for c in range(src.shape[2])], -1)


def fix(x):
    """libjpeg's FIX(x) at SCALEBITS 16"""
    return int(x * 65536 + 0.5)


def bgr_to_ycc(bgr):
    """libjpeg's rgb_ycc_convert (jccolor.c) per pixel: int64 planes Y, Cb, Cr"""
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    y = (fix(.299) * r + fix(.587) * g + fix(.114) * b + (1 << 15)) >> 16
    cb = (-fix(.16874) * r - fix(.33126) * g + fix(.5) * b + (128 << 16) + (1 << 15) - 1) >> 16
    cr = (fix(.5) * r - fix(.41869) * g - fix(.08131) * b + (128 << 16) + (1 << 15) - 1) >> 16
    return y, cb, cr


def h2v2_downsample(c):
    """libjpeg's h2v2_downsample (jcsample.c) of one full-resolution plane: (c00 + c01 + c10 + c11 + bias) >> 2 with bias
    1 on even and 2 on odd output columns (restarting on every row); an odd last column is replicated (expand_right_edge)
    and an odd last row too (expand_bottom_edge, jcprepct.c).  Returns ceil(h/2) x ceil(w/2)."""
    h, w = c.shape
    c = np.pad(c, ((0, h & 1), (0, w & 1)), mode="edge").astype(np.int64)
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    bias = 1 + (np.arange(s.shape[1]) & 1)
    return ((s + bias[None, :]) >> 2).astype(np.uint8)


def bgr_to_ycc420(bgr):
    """The three planes libjpeg hands to its forward DCT for imencode(".jpg", bgr) at 4:2:0:
    (y [h,w], cb [ceil(h/2),ceil(w/2)], cr [ceil(h/2),ceil(w/2)]) uint8."""
    y, cb, cr = bgr_to_ycc(bgr)
    return y.astype(np.uint8), h2v2_downsample(cb), h2v2_downsample(cr)


def mcu_padded(bgr, mcu=16):
    """the frame padded to whole MCUs by replicating its last column and row, as libjpeg's edge expansion does before the
    downsampling: the chroma of the padding then lies in the decoded image's chroma blocks too"""
    h, w = bgr.shape[:2]
    return np.pad(bgr, ((0, -h % mcu), (0, -w % mcu), (0, 0)), mode="edge")
