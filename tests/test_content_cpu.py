"""The content recipes of tests/content_cases.py on the CPU oracles.

* Each recipe still drives the regime it was written for (a later edit must not quietly turn it into easy content).
* The Farneback oracle against live cv2.calcOpticalFlowFarneback, per class and at both test sizes.
* The C TV-L1 oracle against the separately written numpy restatement (oracle/tvl1_numpy.py) on small versions of every
  class, so that the second restatement also covers flat (g <= FLT_EPSILON) pixels, pairs that run into the iteration cap
  and warps whose taps are clamped far outside the image."""
import numpy as np
import pytest

import content_cases as cc
from denseflow_b200 import synth

W, H = cc.SIZE


@pytest.fixture(scope="module")
def tvl1_340(oracle):
    """the oracle's TV-L1 (flow, log) of every class at 340 x 256"""
    return {c: oracle.tvl1_calc(*cc.pair(c, W, H), return_iters=True) for c in cc.CLASSES}


def test_recipes_are_deterministic():
    for c in cc.CLASSES:
        a, b = cc.pair(c, 56, 40)
        a2, b2 = cc.pair(c, 56, 40)
        assert a.dtype == b.dtype == np.uint8 and a.shape == b.shape == (40, 56), c
        assert np.array_equal(a, a2) and np.array_equal(b, b2), c
    s = cc.stream(56, 40)
    assert s.shape == (2 * len(cc.STREAM_CLASSES), 40, 56) and np.array_equal(s, cc.stream(56, 40))
    a, b = cc.case_pair("letterbox_239", 64, 300)
    assert not a[:140].any() and not a[160:].any() and a[140:160].all() and not b[:140].any()


def test_flat_fraction(oracle):
    """share of pixels on the primal step's g <= FLT_EPSILON branch at the finest level at zero flow"""
    frac = {c: cc.flat_fraction(oracle, cc.pair(c, W, H)[1]) for c in ("synth", "letterbox", "pillarbox", "checkerboard", "fade_black")}
    assert frac["synth"] < 1e-3, frac  # 0.04 %: isolated pixels whose two central differences both vanish
    assert frac["letterbox"] > 0.2 and frac["pillarbox"] > 0.2 and frac["checkerboard"] > 0.2, frac
    assert frac["fade_black"] == 1.0, frac


def test_tvl1_regimes(tvl1_340):
    for c in cc.AT_MINIMUM:
        assert (tvl1_340[c][1] == 2).all(), (c, tvl1_340[c][1].tolist())
    for c in cc.AT_CAP:
        assert (tvl1_340[c][1] == 300).all(), (c, tvl1_340[c][1].tolist())
    for c in ("fade_half", "fade_from_black"):  # warp taps clamped far outside the image, quantiser saturated over whole planes
        assert np.abs(tvl1_340[c][0]).max() > W, (c, np.abs(tvl1_340[c][0]).max())
    for c in ("static", "fade_black"):
        assert not tvl1_340[c][0].any(), c
    # the classes the default build must hold to the AEE contract converge somewhere and run into the cap somewhere else
    for c in ("synth", "letterbox", "pillarbox", "clipped", "checkerboard"):
        log = tvl1_340[c][1]
        assert log.min() < 300 and log.max() == 300, (c, log.tolist())
    for c in cc.CLASSES:
        assert np.isfinite(tvl1_340[c][0]).all(), c


# oracle (half-pixel resize convention) against live cv2 at 340 x 256 and 131 x 97: (AEE, max |diff|, max |diff| beyond the
# 8 px border band), each about ten times the larger of the two sizes' measured figure
FARN_CV2 = {
    "synth": (4e-6, 3e-5, 3e-5),
    "letterbox": (7e-6, 2e-3, 2e-3),
    "pillarbox": (4e-6, 5e-4, 5e-4),
    "static": (1e-3, 1.2, 2e-3),
    "fade_half": (4e-6, 3e-5, 2e-5),
    "fade_black": (1.5e-4, 4e-4, 4e-4),
    "fade_from_black": (2e-4, 4e-3, 2e-3),
    "cut": (7e-4, 8e-2, 8e-2),
    "pan": (7e-5, 3e-3, 3e-3),
    "pan_diagonal": (2e-4, 2e-2, 2e-2),
    "clipped": (4e-6, 7e-5, 3e-5),
    "checkerboard": (6e-6, 5e-5, 2e-5),
    "square": (3e-4, 0.4, 6e-4),
    "noise": (2e-6, 7e-6, 7e-6),
}


@pytest.mark.parametrize("size", [cc.SIZE, cc.SMALL], ids=["340x256", "131x97"])
@pytest.mark.parametrize("name", cc.CLASSES)
def test_farneback_oracle_against_opencv(oracle, name, size):
    """The oracle in the half-pixel resize convention against cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 5, 13, 10, 5, 1.1, 0).

    Measured (AEE / max |diff| in px, 340 x 256): 4e-7 / 3e-6 on synth, checkerboard, clipped and fade to half; 1-7e-5 /
    4e-4-8.5e-3 on the cut, both pans and the fades from and to black, where the ill-posed flow is sensitive to the last bit
    of every input; 8e-5 / 0.12 on the static pair and 2-3e-5 / 0.04 on the square.  The static and square figures are border
    figures: beyond the 8 px border band their differences stay below 2e-4 px.  In that band the two implementations
    separate on the border convention of DESIGN §3: CPU OpenCV takes the R1 samples of a displaced position outside the image
    as zero, the oracle clamps them as CUDA OpenCV does (and so does the engine, which is pinned to the oracle)."""
    import cv2
    w, h = size
    a, b = cc.pair(name, w, h)
    mine = oracle.farn_calc(a, b, oracle.farn_params(resize_convention=oracle.RESIZE_HALF_PIXEL))
    live = cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 5, 13, 10, 5, 1.1, 0)
    d = np.hypot(*(mine.astype(np.float64) - live).transpose(2, 0, 1))
    aee_b, max_b, inner_b = FARN_CV2[name]
    assert np.isfinite(mine).all()
    assert synth.aee(mine, live) <= aee_b, (synth.aee(mine, live), aee_b)
    assert d.max() <= max_b, (d.max(), max_b)
    assert d[8:-8, 8:-8].max() <= inner_b, (d[8:-8, 8:-8].max(), inner_b)


@pytest.mark.parametrize("name", cc.CLASSES)
def test_tvl1_c_oracle_agrees_with_numpy_restatement(oracle, name):
    """as tests/test_oracle_cpu.py::test_tvl1_c_oracle_agrees_with_independent_numpy_restatement, at 56 x 40 with 3 scales x 2
    warps x 40 iterations: the same schedule, the flows equal to fp32 rounding (measured: identical on every class)"""
    from oracle import tvl1_numpy as N
    a, b = cc.pair(name, 56, 40)
    prm = oracle.tvl1_params(nscales=3, warps=2, iterations=40)
    fc, lc = oracle.tvl1_calc(a, b, prm, return_iters=True)
    with np.errstate(invalid="ignore", divide="ignore"):  # -rho / g of flat pixels, discarded by the g > eps select
        fn, ln = N.calc(a, b, nscales=3, warps=2, iterations=40)
    assert np.array_equal(lc[:3, :2], ln[:3, :2]), (lc.tolist(), ln.tolist())
    assert np.abs(fc - fn).max() < 5e-4 and synth.aee(fc, fn) < 2e-5
    if name in cc.AT_CAP:
        assert (lc[:3, :2] == 40).all()
    if name in ("letterbox", "pillarbox", "checkerboard", "fade_black"):
        assert cc.flat_fraction(oracle, b) > 0.1
