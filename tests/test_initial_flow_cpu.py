"""`use_initial_flow` in its restatements (tests/tvl1_restate.py, tests/farn_restate.py), before the GPU builds are
pinned to them (tests/test_initial_flow_gpu.py).

* TV-L1: the initial-flow pyramid over the C oracle's building blocks and over oracle/tvl1_numpy.py's agree bit for bit,
  at 1, 5 and 16 levels, small scale steps, and tiny and thin frames whose pyramid stops at 16 pixels; the two whole
  solves from an initial flow agree (equal iteration logs, flows to the fp32 rounding the cold restatements already
  differ by), median filtering on or off.
* A zero initial flow is orc_tvl1_calc and orc_farn_calc bit for bit.
* Farneback with one level (num_levels 0) in OpenCV-CPU's resize convention is live
  cv2.calcOpticalFlowFarneback(..., OPTFLOW_USE_INITIAL_FLOW) within the tolerance of the cold live pin
  (tests/test_oracle_cpu.py).  With more levels CPU OpenCV resizes the initial flow with INTER_AREA, not the CUDA module's
  INTER_LINEAR: that AEE is printed, not asserted."""
import numpy as np
import pytest

import farn_restate as R
import tvl1_restate as T
from denseflow_b200 import synth

F = np.float32


def smooth_field(h, w, seed, amp=2.0):
    """a smooth random flow [H,W,2]: a few low-frequency cosines per channel"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.zeros((h, w, 2))
    for c in range(2):
        for _ in range(3):
            fx, fy, ph = rng.uniform(0.2, 2.0) * np.pi / max(w, 1), rng.uniform(0.2, 2.0) * np.pi / max(h, 1), rng.uniform(0, 2 * np.pi)
            out[..., c] += rng.uniform(-1, 1) * np.cos(fx * x + fy * y + ph)
    return (amp * out / 3).astype(F)


PYRAMIDS = [(96, 80, 1, 0.8), (96, 80, 5, 0.8), (340, 256, 16, 0.8), (340, 256, 16, 0.5), (340, 256, 16, 0.3), (24, 40, 5, 0.8),
            (17, 300, 16, 0.8), (300, 17, 16, 0.8), (16, 16, 5, 0.8), (33, 33, 16, 0.5)]


@pytest.mark.parametrize("w,h,nscales,step", PYRAMIDS)
def test_initial_flow_pyramids_agree_bit_for_bit(oracle, w, h, nscales, step):
    init = smooth_field(h, w, w * 7 + h, amp=5.0)
    lv = oracle.tvl1_level_sizes(w, h, oracle.tvl1_params(nscales=nscales, scale_step=step))
    c1, c2 = T.tvl1_init_pyramid(init, lv, step)
    n1, n2 = T.numpy_init_pyramid(init, nscales, step)
    assert [p.shape[::-1] for p in c1] == list(lv) == [p.shape[::-1] for p in n1]
    assert lv[-1][0] >= 16 and lv[-1][1] >= 16 or len(lv) == 1
    for s in range(len(lv)):
        for c, n in ((c1[s], n1[s]), (c2[s], n2[s])):
            assert np.array_equal(c.view(np.int32), n.view(np.int32)), (s, lv[s])
    assert np.array_equal(c1[0], init[..., 0]) and np.array_equal(c2[0], init[..., 1])


CASES = [dict(nscales=3, warps=3, iterations=60), dict(nscales=1, warps=3, iterations=40), dict(nscales=5, warps=2, iterations=30),
         dict(nscales=16, warps=1, iterations=10, scale_step=0.5), dict(nscales=3, warps=3, iterations=60, median_filtering=3,
                                                                            median_interval=7),
         dict(nscales=3, warps=2, iterations=40, median_filtering=5, median_interval=5)]


def _ids(cases):
    return ["-".join("%s%g" % (k, v) for k, v in c.items()) for c in cases]


def _numpy_kw(kw):
    return {("lam" if k == "lambda_" else k): v for k, v in kw.items()}


@pytest.mark.parametrize("kw", CASES, ids=_ids(CASES))
@pytest.mark.parametrize("start", ["smooth", "past_bound", "cold_flow"])
def test_two_tvl1_restatements_agree_from_an_initial_flow(oracle, kw, start):
    a, b, _ = synth.pair(80, 96, 6)
    init = {"smooth": lambda: smooth_field(80, 96, 1),
            "past_bound": lambda: smooth_field(80, 96, 2, amp=60.0),
            "cold_flow": lambda: T.tvl1_calc(a, b, **kw)[0]}[start]()
    fc, lc, _ = T.tvl1_calc(a, b, init=init, **kw)
    fn, ln = T.numpy_calc(a, b, init=init, **_numpy_kw(kw))
    assert np.array_equal(lc, ln), (lc.tolist(), ln.tolist())
    assert np.isfinite(fc).all()
    assert np.abs(fc - fn).max() < 5e-4 and synth.aee(fc, fn) < 2e-5
    cold = T.tvl1_calc(a, b, **kw)[0]
    assert not np.array_equal(fc, cold), "the initial flow did not change the result"


@pytest.mark.parametrize("kw", [dict(nscales=3, warps=3, iterations=60), dict(nscales=5, warps=2, iterations=30, median_filtering=3)],
                         ids=["plain", "median"])
def test_zero_initial_flow_is_the_cold_oracle(oracle, kw):
    a, b, _ = synth.pair(80, 96, 6)
    zero = np.zeros((80, 96, 2), F)
    f0, l0, e0 = T.tvl1_calc(a, b, init=zero, **kw)
    fn, ln, en = T.tvl1_calc(a, b, **kw)
    assert np.array_equal(f0.view(np.int32), fn.view(np.int32)) and np.array_equal(l0, ln) and np.array_equal(e0, en)
    if "median_filtering" not in kw:
        ref, log = oracle.tvl1_calc(a, b, oracle.tvl1_params(**kw), return_iters=True)
        assert np.array_equal(f0.view(np.int32), ref.view(np.int32)) and np.array_equal(l0, log)
    g0, m0 = T.numpy_calc(a, b, init=zero, **_numpy_kw(kw))
    gn, mn = T.numpy_calc(a, b, **_numpy_kw(kw))
    assert np.array_equal(g0.view(np.int32), gn.view(np.int32)) and np.array_equal(m0, mn)


@pytest.mark.parametrize("num_levels", [0, 2, 5])
def test_farneback_restatement_zero_start_is_orc_farn_calc(oracle, num_levels):
    a, b, _ = synth.pair(96, 128, 3)
    p = oracle.farn_params(num_levels=num_levels)
    ref = oracle.farn_calc(a, b, p)
    for init in (None, np.zeros((96, 128, 2), F)):
        got = R.farn_calc(a, b, init=init, params=p)
        assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    assert not np.array_equal(R.farn_calc(a, b, init=smooth_field(96, 128, 4), params=p), ref)


@pytest.mark.parametrize("hw", [(256, 256, 0), (256, 340, 100)])
def test_farneback_one_level_matches_live_opencv_with_initial_flow(oracle, hw):
    cv2 = pytest.importorskip("cv2")
    h, w, seed = hw
    a, b, _ = synth.pair(h, w, seed)
    init = smooth_field(h, w, seed + 1, amp=8.0)
    p = oracle.farn_params(num_levels=0, resize_convention=oracle.RESIZE_HALF_PIXEL)
    mine = R.farn_calc(a, b, init=init, params=p)
    live = cv2.calcOpticalFlowFarneback(a, b, init.copy(), 0.5, 0, 13, 10, 5, 1.1, cv2.OPTFLOW_USE_INITIAL_FLOW)
    assert synth.aee(mine, live) < 5e-6
    cold = cv2.calcOpticalFlowFarneback(a, b, None, 0.5, 0, 13, 10, 5, 1.1, 0)
    assert np.abs(live - cold).max() > 1e-2  # the initial flow is really used
    # more levels: CPU OpenCV resizes the initial flow with INTER_AREA, the CUDA module (and this contract) with INTER_LINEAR
    multi = R.farn_calc(a, b, init=init, params=oracle.farn_params(resize_convention=oracle.RESIZE_HALF_PIXEL))
    live5 = cv2.calcOpticalFlowFarneback(a, b, init.copy(), 0.5, 5, 13, 10, 5, 1.1, cv2.OPTFLOW_USE_INITIAL_FLOW)
    print("farneback %dx%d, 5 levels from an initial flow: AEE vs cv2 (INTER_AREA start) = %.3e px" % (w, h, synth.aee(multi, live5)))
