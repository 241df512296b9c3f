"""The optional median filtering of the TV-L1 flow (DESIGN §4.3) in its two restatements (tests/tvl1_restate.py), before
the GPU builds are pinned to them (tests/test_tvl1_median_gpu.py).

* M_k: the key-ordered median and the by-value median equal cv2.medianBlur at k = 3 and 5.  cv2 is compared by value: the
  sign of a zero it returns depends on its sorting network, while the contract orders -0 below +0, which both
  restatements follow bit for bit.
* The flow over the C oracle's building blocks and the one over oracle/tvl1_numpy.py's agree with the median on: equal
  iteration logs, flows within the tolerance of the off-default comparison in tests/test_params_cpu.py.
* With median_filtering 0 or 1 the first is orc_tvl1_calc bit for bit (flow, log and every convergence check to rounding), and the
  median does change the flow."""
import itertools
import os

import cv2
import numpy as np
import pytest

import tvl1_restate as T
from denseflow_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMALL = [(w, h) for w in range(1, 9) for h in range(1, 9)]
EDGES = [(w, h) for w in (15, 16, 17) for h in (15, 16, 17)] + [(1, 40), (40, 1), (1, 333), (333, 1), (2, 77), (77, 2)]


def _planes(w, h, seed):
    rng = np.random.default_rng(seed)
    return [("iid", (rng.standard_normal((h, w)) * 3).astype(np.float32)),
            ("ties", rng.choice(np.float32([-1.5, 0.0, 0.25, 2.0]), (h, w)).astype(np.float32)),
            ("constant", np.full((h, w), np.float32(-0.75)))]


def _same_values(got, want, what):
    bad = got != want
    assert not bad.any(), "%s: %d of %d differ, first at %s: %r vs %r" % (what, bad.sum(), bad.size, tuple(np.argwhere(bad)[0]),
                                                                          got[tuple(np.argwhere(bad)[0])], want[tuple(np.argwhere(bad)[0])])


@pytest.mark.parametrize("k", [3, 5])
def test_median_blur_equals_cv2(k):
    for j, (w, h) in enumerate(SMALL + EDGES + [(340, 256)]):
        for name, a in _planes(w, h, 100 * k + j):
            want = cv2.medianBlur(a, k)
            what = "%dx%d %s k %d" % (w, h, name, k)
            c = T.median_blur(a, k)
            _same_values(c, want, what + " by key")
            n = T.median_blur_by_value(a, k)
            _same_values(n, want, what + " by value")
            assert np.array_equal(c.view(np.int32), n.view(np.int32)), what + ": the two restatements differ in a bit"


@pytest.mark.parametrize("k", [3, 5])
def test_median_blur_1080p_equals_cv2(k):
    a = (np.random.default_rng(k).standard_normal((1080, 1920)) * 4).astype(np.float32)
    _same_values(T.median_blur(a, k), cv2.medianBlur(a, k), "1920x1080 k %d" % k)


def _rule(a, k):
    """the contract itself, pixel by pixel: the element of rank (k*k - 1) / 2 of the replicate-padded window sorted by
    (value, +0 above -0)"""
    h, w = a.shape
    r, m = k // 2, (k * k - 1) // 2
    out = np.empty_like(a)
    for y, x in itertools.product(range(h), range(w)):
        win = [a[min(max(y + dy, 0), h - 1), min(max(x + dx, 0), w - 1)] for dy in range(-r, r + 1) for dx in range(-r, r + 1)]
        out[y, x] = sorted(win, key=lambda v: (float(v), not np.signbit(v)))[m]
    return out


@pytest.mark.parametrize("k", [3, 5])
def test_signed_zeros_follow_the_contract(k):
    rng = np.random.default_rng(k)
    for j, (w, h) in enumerate([(1, 1), (3, 2), (7, 5), (24, 19)]):
        a = rng.choice(np.float32([-0.0, 0.0, -0.0, 0.0, 1.0, -1.0]), (h, w)).astype(np.float32)
        want = _rule(a, k)
        for name, got in (("by key", T.median_blur(a, k)), ("by value", T.median_blur_by_value(a, k))):
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), "%dx%d k %d %s: the sign of a zero differs" % (w, h, k, name)
        if w * h > 100:  # the case exists: zeros of both signs in the result
            z = want[want == 0]
            assert np.signbit(z).any() and (~np.signbit(z)).any()


# (median_filtering, median_interval, other parameters): k 3 / 5, I 1 / 2 / 7 / 30 / 300, epsilon 0 / 0.01 / 1.0,
# iterations 1 / 2 / 3 / 60, small pyramids
BASE = dict(nscales=3, warps=3, iterations=60)
CASES = [(3, 1, {}), (5, 1, {}), (3, 2, {}), (5, 2, dict(epsilon=0.0, iterations=9)), (3, 7, {}), (5, 7, dict(epsilon=1.0)),
         (3, 30, {}), (5, 30, dict(epsilon=0.0)), (3, 300, {}), (5, 300, dict(iterations=1)), (3, 1, dict(iterations=2)),
         (5, 2, dict(iterations=3)), (3, 7, dict(epsilon=0.0, nscales=1, warps=2)), (5, 30, dict(nscales=2, warps=5)),
         (3, 2, dict(epsilon=1.0, warps=1))]


def _ids(cases):
    return ["k%d-I%d%s" % (k, i, "".join("-%s%g" % kv for kv in p.items())) for k, i, p in cases]


@pytest.mark.parametrize("case", CASES, ids=_ids(CASES))
def test_c_oracle_agrees_with_numpy_restatement(oracle, case):
    k, interval, prm = case
    kw = dict(BASE, **prm)
    a, b, _ = synth.pair(80, 96, 6)
    fc, lc, _ = T.tvl1_calc(a, b, median_filtering=k, median_interval=interval, **kw)
    fn, ln = T.numpy_calc(a, b, median_filtering=k, median_interval=interval, **kw)
    assert np.array_equal(lc, ln), (lc.tolist(), ln.tolist())
    if prm.get("epsilon") == 1.0:  # every warp converges at its first check
        n = len(oracle.tvl1_level_sizes(96, 80, oracle.tvl1_params(nscales=kw["nscales"])))
        assert (lc[:n] == 2).all()
    assert np.isfinite(fc).all()
    assert np.abs(fc - fn).max() < 5e-4 and synth.aee(fc, fn) < 2e-5
    off = oracle.tvl1_calc(a, b, oracle.tvl1_params(**kw))  # the C oracle: no median
    assert (fc != off).any(), "the median did not change the flow"


def _same_checks(got, want):
    """the same convergence checks; the error sums equal to rounding: the oracle adds its OpenMP threads' partial sums in
    an order that changes from run to run"""
    return got.shape == want.shape and np.array_equal(got[:, 1], want[:, 1]) and bool(
        np.all(np.abs(got[:, 0] - want[:, 0]) <= 1e-12 * np.abs(want[:, 0])))


def test_median_off_is_the_c_oracle(oracle):
    """0 and 1 mean off at any interval: the restatement over the building blocks is orc_tvl1_calc bit for bit (flow, log
    and every convergence check), here and away from the defaults, and the frozen regression fixture holds"""
    gold = np.load(os.path.join(GOLD, "tvl1_oracle_256.npz"))
    a, b, _ = synth.pair(256, 256, 0)
    ref, log, errs = oracle.tvl1_calc(a, b, return_iters=True, return_errors=True)
    assert np.array_equal(log, gold["iters"])
    assert np.array_equal(ref[::4, ::4], gold["flow_s4"])
    for mf, interval in ((0, 30), (1, 30), (0, 1), (1, 7)):
        f, lg, e = T.tvl1_calc(a, b, median_filtering=mf, median_interval=interval)
        assert np.array_equal(f.view(np.int32), ref.view(np.int32)) and np.array_equal(lg, log), (mf, interval)
        assert _same_checks(e, errs), (mf, interval)
    a, b, _ = synth.pair(80, 96, 6)
    for kw in (dict(BASE), dict(BASE, epsilon=0.0, iterations=9), dict(BASE, epsilon=1.0), dict(tau=0.5, theta=0.05, nscales=2)):
        ref, log, errs = oracle.tvl1_calc(a, b, oracle.tvl1_params(**kw), return_iters=True, return_errors=True)
        f, lg, e = T.tvl1_calc(a, b, median_filtering=0, median_interval=30, **kw)
        assert np.array_equal(f.view(np.int32), ref.view(np.int32)) and np.array_equal(lg, log) and _same_checks(e, errs), kw


def test_restatements_refuse_bad_median_parameters():
    a, b, _ = synth.pair(32, 32, 1)
    for mf, interval in ((2, 30), (4, 30), (7, 30), (-1, 30), (3, 0), (5, -4)):
        with pytest.raises(ValueError):
            T.tvl1_calc(a, b, median_filtering=mf, median_interval=interval)
        with pytest.raises(ValueError):
            T.numpy_calc(a, b, median_filtering=mf, median_interval=interval)
    for k in (1, 4, 7):
        with pytest.raises(ValueError):
            T.median_blur(np.zeros((4, 4), np.float32), k)
