"""Images that drive libjpeg's entropy coder into its edge cases, found with the restatement (tests/jpeg_encode_restate.py)
and checked there: the CPU test asserts each case really hits its edge, the GPU test encodes them."""
import numpy as np

import jpeg_encode_restate as E


def _basis(z, amp=127):
    """an 8 x 8 block holding DC 0 plus one strong cosine basis function at zig-zag index z"""
    k = int(E.ZIGZAG[z])
    u, v = k % 8, k // 8
    x = np.arange(8)
    f = np.outer(np.cos((2 * x + 1) * v * np.pi / 16), np.cos((2 * x + 1) * u * np.pi / 16))
    return np.clip(np.round(128 + amp * f / np.abs(f).max()), 0, 255).astype(np.uint8)


def zz_coefficients(img, q):
    coef, _ = E.coefficients(img, q)
    return coef[:, E.ZIGZAG]


def run_cases():
    """(name, image, quality, zig-zag index of the block's only AC coefficient): at quality 1 every quantiser step is
    255, so one strong basis function leaves exactly one nonzero AC coefficient"""
    out = []
    for run in (15, 16, 17, 31, 32):
        out.append(("run%d_before_nonzero" % run, _basis(run + 1), 1, run + 1))
        out.append(("run%d_before_end" % run, _basis(63 - run), 1, 63 - run))
    out.append(("last_coefficient_nonzero", _basis(63), 1, 63))
    return out


def dc_category11():
    """alternating black and white blocks at quality 100: DC differences of +-2040 (category 11)"""
    bx = (np.arange(32)[None, :] // 8 + np.arange(16)[:, None] // 8) & 1
    return (bx * 255).astype(np.uint8)


def ff_flush_case():
    """an 8 x 8 image whose final entropy byte, padded with 1-bits, is 0xFF (stuffed): the first seed that gives one"""
    for seed in range(20000):
        img = np.random.default_rng(seed).integers(0, 256, (8, 8), dtype=np.uint8)
        coef, comp = E.coefficients(img, 50)
        data, nbits = E.entropy(coef, comp, with_bits=True)
        if nbits % 8 and data.endswith(b"\xff\x00"):
            return img
    raise AssertionError("no seed found")


def entropy_cases():
    """(name, image, quality) of every entropy-coder edge case"""
    cases = [(n, img, q) for n, img, q, _ in run_cases()]
    cases.append(("dc_category11", dc_category11(), 100))
    noise = np.random.default_rng(1).integers(0, 256, (24, 40), dtype=np.uint8)
    cases.append(("ff_bytes", noise, 100))
    cases.append(("ff_flush", ff_flush_case(), 50))
    cases.append(("ff_bytes_colour", np.random.default_rng(2).integers(0, 256, (24, 40, 3), dtype=np.uint8), 100))
    return cases
