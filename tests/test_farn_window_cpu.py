"""Farneback's Gaussian window and fast pyramids (SURVEY B.7) restated over the oracle's building blocks
(tests/farn_restate.py), pinned without a GPU:

* with both options off the restatement is orc_farn_calc bit for bit, so it adds nothing to the default path;
* with CPU OpenCV's half-pixel resize the Gaussian window matches live cv2.calcOpticalFlowFarneback(...,
  OPTFLOW_FARNEBACK_GAUSSIAN), cold and warm-started;
* its pyrDown is within a stated fp32 bound of cv2.pyrDown, and the pyrDown level sizes and count follow the contract;
* its window weights are cv2.getGaussianKernel(13, 1.8f) within one fp32 rounding."""
import cv2
import numpy as np
import pytest

import farn_restate as R
from denseflow_b200 import synth

GAUSS = cv2.OPTFLOW_FARNEBACK_GAUSSIAN
# AEE of the restatement (half-pixel resize) against live cv2 with the Gaussian window; measured 7.6e-7 px at 256 x 256
# and 8.7e-7 px at 340 x 256: the window weights and the resize are CPU OpenCV's to the last bits or nearly
AEE_CV2 = 5e-6


@pytest.fixture(autouse=True)
def _one_thread(oracle):
    # these planes are small: the oracle's OpenMP loops are fastest on one thread here
    oracle.lib().orc_set_num_threads(1)
    yield
    oracle.lib().orc_set_num_threads(min(8, oracle.usable_cores()))


def _aee(a, b):
    return float(np.hypot(*(np.asarray(a, np.float64) - b).transpose(2, 0, 1)).mean())


@pytest.mark.parametrize("shape,params", [((256, 256), {}), ((256, 340), {}), ((97, 131), {"num_levels": 3}),
                                          ((97, 131), {"num_iters": 2, "poly_sigma": 1.5})])
def test_options_off_is_the_oracle(oracle, shape, params):
    h, w = shape
    a, b, _ = synth.pair(h, w, 1)
    p = oracle.farn_params(**params)
    assert np.array_equal(R.farn_calc(a, b, params=p), oracle.farn_calc(a, b, p))


@pytest.mark.parametrize("shape,levels", [((256, 256), 5), ((256, 340), 5), ((256, 256), 2), ((256, 340), 1)])
def test_gaussian_window_matches_cv2(oracle, shape, levels):
    h, w = shape
    a, b, _ = synth.pair(h, w, 0)
    got = R.farn_calc(a, b, params=oracle.farn_params(num_levels=levels, resize_convention=oracle.RESIZE_HALF_PIXEL),
                      gaussian_window=1)
    want = cv2.calcOpticalFlowFarneback(a, b, None, 0.5, levels, 13, 10, 5, 1.1, GAUSS)
    aee = _aee(got, want)
    print("%dx%d levels %d: AEE %.3g px" % (w, h, levels, aee))
    assert aee <= AEE_CV2
    # the window changes the flow: the box would not pass for it
    assert _aee(cv2.calcOpticalFlowFarneback(a, b, None, 0.5, levels, 13, 10, 5, 1.1, 0), want) > 10 * AEE_CV2


@pytest.mark.parametrize("shape", [(256, 256), (256, 340)])
def test_gaussian_window_warm_start_matches_cv2(oracle, shape):
    """OPTFLOW_USE_INITIAL_FLOW at num_levels 0: cv2 resizes the start with INTER_AREA, which at one level is the identity"""
    h, w = shape
    a, b, _ = synth.pair(h, w, 2)
    init = np.ascontiguousarray(cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 5, 13, 10, 5, 1.1, 0) * np.float32(0.8))
    p = oracle.farn_params(num_levels=0, resize_convention=oracle.RESIZE_HALF_PIXEL)
    got = R.farn_calc(a, b, init=init, params=p, gaussian_window=1)
    want = cv2.calcOpticalFlowFarneback(a, b, init.copy(), 0.5, 0, 13, 10, 5, 1.1, GAUSS | cv2.OPTFLOW_USE_INITIAL_FLOW)
    aee = _aee(got, want)
    print("%dx%d warm start: AEE %.3g px" % (w, h, aee))
    assert aee <= AEE_CV2
    cold = cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 0, 13, 10, 5, 1.1, GAUSS)
    assert _aee(cold, want) > 10 * AEE_CV2


def test_gaussian_weights_match_cv2():
    g = R.gauss_weights()
    want = cv2.getGaussianKernel(13, float(np.float32(6) * np.float32(0.3)), cv2.CV_32F).ravel()
    assert np.all(np.abs(g - want[6:]) <= np.spacing(want[6:])), (g, want[6:])
    assert np.array_equal(want[6:], want[6::-1])


@pytest.mark.parametrize("shape", [(1, 1), (1, 2), (2, 1), (2, 3), (2, 2), (3, 3), (5, 7), (7, 5), (45, 64), (48, 64),
                                   (97, 131), (256, 340), (255, 1)])
def test_pyr_down_matches_cv2(shape):
    """|restatement - cv2.pyrDown| <= 2^-20 x the pyrDown of |image|: 16 fp32 roundings of the largest term's size, for two
    evaluation orders of a 25-tap filter with dyadic weights"""
    h, w = shape
    img = np.random.default_rng(h * 1000 + w).uniform(-300, 300, (h, w)).astype(np.float32)
    got, want = R.pyr_down(img), cv2.pyrDown(img)
    assert got.shape == want.shape == ((h + 1) // 2, (w + 1) // 2)
    bound = 2.0 ** -20 * R.pyr_down(np.abs(img)).astype(np.float64)
    diff = np.abs(got.astype(np.float64) - want)
    assert np.all(diff <= bound), (diff.max(), bound[diff > bound][:3])


def test_pyr_down_level_sizes(oracle):
    # B.1's count, the chain's sizes: one pixel larger than cvRound's where a level has an odd side
    assert R.level_sizes(340, 256, fast_pyramids=1) == [(43, 32), (85, 64), (170, 128), (340, 256)]
    assert R.level_sizes(340, 256) == [(42, 32), (85, 64), (170, 128), (340, 256)]
    assert R.level_sizes(131, 97, fast_pyramids=1) == [(66, 49), (131, 97)]
    assert R.level_sizes(131, 97) == [(66, 48), (131, 97)]
    assert R.pyr_down(np.zeros((45, 90), np.float32)).shape == (23, 45)  # cvRound(45 * 0.5) is 22
    for (w, h) in [(1920, 1080), (1280, 720), (455, 256), (340, 256), (33, 49), (5, 7), (1, 200)]:
        for levels in (0, 1, 3, 5):
            p = oracle.farn_params(num_levels=levels)
            fast, b1 = R.level_sizes(w, h, p, 1), R.level_sizes(w, h, p, 0)
            assert len(fast) == len(b1) and fast[-1] == (w, h)
            chain = [np.zeros((h, w), np.float32)]
            for _ in range(len(fast) - 1):
                chain.append(cv2.pyrDown(chain[-1]))
            assert fast == [(c.shape[1], c.shape[0]) for c in chain[::-1]]
            assert all(fw >= bw and fh >= bh for (fw, fh), (bw, bh) in zip(fast, b1))
