"""The TV-L1 illumination term (`gamma`; SURVEY.md A.8) in its two restatements (tests/tvl1_restate.py), before the GPU
builds are pinned to them (tests/test_tvl1_gamma_gpu.py).

* At gamma = 0 each restatement is its oracle bit for bit: flows and iteration logs (and the C one every convergence check).
* At gamma > 0 the two agree as closely as the cold restatements do, with equal iteration logs, also with the median and a
  warm start.
* On a pair whose second frame is brighter the term does something: u3 is nonzero and the flow differs from gamma = 0.
* The restatements refuse what the handles refuse.
* The accuracy table of scripts/gamma_quality.py is printed, not asserted."""
import numpy as np
import pytest

import tvl1_restate as T
from denseflow_b200 import synth

BASE = dict(nscales=3, warps=3, iterations=60)


def _brighter(b, gain=1.1, offset=8.0):
    return np.clip(np.rint(b.astype(np.float64) * gain + offset), 0, 255).astype(np.uint8)


def _same_checks(got, want):
    """the oracle adds its OpenMP threads' partial sums in an order that changes from run to run"""
    return got.shape == want.shape and np.array_equal(got[:, 1], want[:, 1]) and bool(
        np.all(np.abs(got[:, 0] - want[:, 0]) <= 1e-12 * np.abs(want[:, 0])))


@pytest.mark.parametrize("kw", [{}, dict(BASE), dict(BASE, epsilon=0.0, iterations=9), dict(tau=0.5, theta=0.05, nscales=2)])
def test_gamma_zero_is_each_oracle(oracle, kw):
    from oracle import tvl1_numpy as N
    h, w = (256, 256) if not kw else (80, 96)
    a, b, _ = synth.pair(h, w, 0 if not kw else 6)
    ref, log, errs = oracle.tvl1_calc(a, b, oracle.tvl1_params(**kw), return_iters=True, return_errors=True)
    f, lg, e = T.tvl1_calc(a, b, gamma=0.0, **kw)
    assert np.array_equal(f.view(np.int32), ref.view(np.int32)) and np.array_equal(lg, log) and _same_checks(e, errs)
    nkw = {("lam" if k == "lambda" else k): v for k, v in kw.items()}
    nref, nlog = N.calc(a, b, **nkw)
    fn, ln = T.numpy_calc(a, b, gamma=0.0, **nkw)
    assert np.array_equal(fn.view(np.int32), nref.view(np.int32)) and np.array_equal(ln, nlog)


# (gamma, brighter second frame, other parameters)
CASES = [(0.1, True, {}), (1.0, True, {}), (0.5, False, {}), (1.0, True, dict(epsilon=0.0, iterations=9)),
         (1.0, True, dict(epsilon=1.0)), (3.0, True, dict(nscales=1, warps=2)), (0.25, True, dict(tau=0.5, theta=0.05)),
         (1.0, True, dict(median_filtering=3, median_interval=7)), (1.0, True, dict(warm=True))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_restatements_agree(oracle, case):
    gamma, bright, prm = CASES[case]
    prm = dict(prm)
    kw = dict(BASE, **prm)
    a, b, gt = synth.pair(80, 96, 6)
    if bright:
        b = _brighter(b)
    init = None
    if kw.pop("warm", False):
        init = (gt * 0.5).astype(np.float32)
    fc, lc, _ = T.tvl1_calc(a, b, gamma=gamma, init=init, **kw)
    fn, ln = T.numpy_calc(a, b, gamma=gamma, init=init, **kw)
    assert np.array_equal(lc, ln), (lc.tolist(), ln.tolist())
    assert np.isfinite(fc).all()
    # the tolerance of the cold restatements' comparison (tests/test_tvl1_median_cpu.py)
    assert np.abs(fc - fn).max() < 5e-4 and synth.aee(fc, fn) < 2e-5


@pytest.mark.parametrize("gamma", [0.1, 1.0])
def test_brightness_change_moves_u3_and_the_flow(gamma):
    a, b, gt = synth.pair(80, 96, 2)
    b = _brighter(b, 1.15, 10.0)
    f, _, _, u3 = T.tvl1_calc(a, b, gamma=gamma, return_u3=True, **BASE)
    f0 = T.tvl1_calc(a, b, gamma=0.0, **BASE)[0]
    assert np.abs(u3).max() > 0.1 and np.isfinite(u3).all()
    assert (f != f0).any()
    if gamma == 1.0:  # the term absorbs the brightness change that gamma = 0 reads as motion
        assert synth.aee(f, gt) < synth.aee(f0, gt)


def test_restatements_refuse_bad_gamma():
    a, b, _ = synth.pair(32, 32, 1)
    for g in (-0.5, -1e-9, float("nan"), float("inf"), float("-inf")):
        with pytest.raises(ValueError):
            T.tvl1_calc(a, b, gamma=g)
        with pytest.raises(ValueError):
            T.numpy_calc(a, b, gamma=g)


def test_print_quality_table():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "scripts", "gamma_quality.py"), "--size", "96", "--seeds", "0"],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("shape", [(1, 1), (5, 3), (37, 53), (128, 131)])
def test_gamma_steps_at_zero_are_the_oracle_steps(oracle, shape):
    """the restatement's own primal step, run with gamma = 0 and u3 = p31 = p32 = 0, is orc_tvl1_estimate_u bit for bit (its
    dual step is the oracle's by construction)"""
    h, w = shape
    rng = np.random.default_rng(h * 131 + w)
    ix = (rng.standard_normal((h, w)) * 8).astype(np.float32)
    iy = (rng.standard_normal((h, w)) * 8).astype(np.float32)
    ix[::5, ::3] = 0
    iy[::5, ::3] = 0  # grad <= eps
    grad = (ix * ix + iy * iy).astype(np.float32)
    rho_c = (rng.standard_normal((h, w)) * 20).astype(np.float32)
    p = [rng.uniform(-1, 1, (h, w)).astype(np.float32) for _ in range(4)]
    u1, u2 = (rng.standard_normal((h, w)).astype(np.float32) for _ in range(2))
    zero = np.zeros((h, w), np.float32)
    l_t, theta = np.float32(0.15 * 0.3), np.float32(0.3)
    n1, n2, n3, e = T.estimate_u_gamma(ix, iy, grad, rho_c, *p, zero, zero, u1, u2, zero, l_t, theta, 0.0)
    r1, r2 = u1.copy(), u2.copy()
    er = oracle.lib().orc_tvl1_estimate_u(ix, iy, grad, rho_c, *p, r1, r2, w, h, l_t, theta, 1)
    assert np.array_equal(n1.view(np.int32), r1.view(np.int32)) and np.array_equal(n2.view(np.int32), r2.view(np.int32))
    assert not n3.any() and abs(e - er) <= 1e-12 * abs(er)
