"""Writes tests/golden/jpeg_encode_cases.npz: a few gray and BGR images, their qualities and their
`cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q])` bytes, so the exact JPEG encoder tests pin the bytes independently of
the cv2 present where they run.  Run from the repository root:
    python tests/golden/make_jpeg_encode_golden.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import jpeg_encode_cases as JC  # noqa: E402


def images():
    rng = np.random.default_rng(2024)
    yy, xx = np.mgrid[0:37, 0:53]
    smooth = (128 + 90 * np.sin(xx / 6.0) * np.cos(yy / 4.0)).astype(np.uint8)
    out = [("gray_noise_17x9_q95", rng.integers(0, 256, (9, 17), dtype=np.uint8), 95),
           ("gray_smooth_53x37_q75", smooth, 75),
           ("gray_constant_33x31_q1", np.full((31, 33), 7, np.uint8), 1),
           ("bgr_noise_17x9_q95", rng.integers(0, 256, (9, 17, 3), dtype=np.uint8), 95),
           ("bgr_smooth_53x37_q50", np.stack([smooth, 255 - smooth, np.roll(smooth, 5, 1)], -1), 50),
           ("bgr_noise_33x31_q100", rng.integers(0, 256, (31, 33, 3), dtype=np.uint8), 100),
           ("bgr_constant_1x1_q95", np.full((1, 1, 3), 90, np.uint8), 95)]
    out += [(n, img, q) for n, img, q in JC.entropy_cases()]
    return out


def main():
    arrays = {"cv2_version": np.array(cv2.__version__)}
    for name, img, q in images():
        arrays["img_" + name] = img
        arrays["q_" + name] = np.array(q)
        arrays["jpg_" + name] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].reshape(-1)
    np.savez_compressed(os.path.join(HERE, "jpeg_encode_cases.npz"), **arrays)


if __name__ == "__main__":
    main()
