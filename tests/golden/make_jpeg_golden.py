"""Writes tests/golden/jpeg_decode_cases.npz: JPEG files and their `cv2.imdecode(buf, IMREAD_COLOR)` pixels, so the GPU
decoder tests pin the pixels independently of the cv2 present where they run.  Run from the repository root:
    python tests/golden/make_jpeg_golden.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_cases as J  # noqa: E402


def cases():
    out = []
    for samp in J.SAMPLINGS:
        out.append(J.encode(J.image("noise", 13, 11), samp, 100))
        out.append(J.encode(J.image("smooth", 45, 61), samp, 95, restart=7))
    out.append(J.encode(J.image("smooth", 48, 96), "420", 95))
    out.append(J.encode(J.image("noise", 64, 80), "422", 95, optimize=True))
    out.append(J.encode(J.image("smooth", 40, 3), "420", 50, luma=90, chroma=30))
    out += list(J.pillow_files().values())
    return out


def main():
    arrays = {"cv2_version": np.array(cv2.__version__)}
    cs = cases()
    arrays["n"] = np.array(len(cs))
    for i, b in enumerate(cs):
        arrays["jpg%d" % i] = np.frombuffer(b, np.uint8)
        arrays["bgr%d" % i] = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    np.savez_compressed(os.path.join(HERE, "jpeg_decode_cases.npz"), **arrays)


if __name__ == "__main__":
    main()
