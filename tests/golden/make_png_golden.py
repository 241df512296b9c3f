"""Writes tests/golden/png_imencode_cases.npz: a few images and their `cv2.imencode(".png")` bytes, so the PNG encoder tests
pin the bytes independently of the zlib present where they run.  Run from the repository root:
    python tests/golden/make_png_golden.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import png_cases as PC  # noqa: E402

CASES = [("noise", 5, 3), ("smooth", 64, 96), ("mixed", 45, 80), ("constant", 9, 1), ("literal", 129, 42), ("ramp", 6, 100),
         ("run259", 1, 0)]


def build(kind, h, w):
    if kind == "literal":
        return PC.literal_noise(h, w)
    if kind == "ramp":
        return PC.ramp(h, w)
    if kind.startswith("run"):
        return PC.run_image(int(kind[3:]))
    return PC.image(kind, h, w)


def main():
    arrays = {"cv2_version": np.array(cv2.__version__)}
    for i, (kind, h, w) in enumerate(CASES):
        img = build(kind, h, w)
        ok, png = cv2.imencode(".png", img)
        assert ok
        arrays["img%d" % i] = img
        arrays["png%d" % i] = png.ravel()
    np.savez_compressed(os.path.join(HERE, "png_imencode_cases.npz"), **arrays)


if __name__ == "__main__":
    main()
