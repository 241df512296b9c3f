"""The TV-L1 oracle away from the create() defaults, before the GPU builds are pinned to it there (tests/test_params_gpu.py).

* The C oracle and the independent numpy restatement (oracle/tvl1_numpy.py) give the same iteration schedule and flows
  equal to fp32 rounding at other tau, lambda, theta, scale_step, nscales, warps, epsilon and iterations.
* orc_tvl1_level_sizes gives known answers at scale steps 0.5 and 0.3 and at the 16-level capacity.
* The float64 bounds of tests/tvl1_ref64.py hold the oracle's building blocks at other l_t, taut, theta and upsample factors,
  so the default build can be held to them there."""
import numpy as np
import pytest

import tvl1_ref64 as r64
from denseflow_b200 import synth
from test_tvl1_reference_cpu import _within
from tvl1_cases import chunk_inputs

# small pyramids and iteration caps keep the numpy restatement's runs near a second each
BASE = dict(nscales=3, warps=3, iterations=60)
OFF_DEFAULTS = [dict(tau=0.1), dict(tau=0.5), dict(lambda_=0.0), dict(lambda_=0.05), dict(lambda_=1.0), dict(theta=0.05),
                dict(theta=1.0), dict(scale_step=0.3, nscales=5), dict(scale_step=0.5, nscales=5), dict(scale_step=0.7, nscales=5),
                dict(nscales=16, warps=1, iterations=10), dict(warps=16, nscales=2, iterations=8), dict(epsilon=1.0, warps=5),
                dict(iterations=1), dict(iterations=2), dict(iterations=3), dict(theta=1.0, scale_step=0.5, nscales=5),
                dict(tau=0.5, theta=0.05, lambda_=1.0)]


def _ids(cases):
    return ["-".join("%s%g" % (k.rstrip("_"), v) for k, v in c.items()) for c in cases]


@pytest.mark.parametrize("prm", OFF_DEFAULTS, ids=_ids(OFF_DEFAULTS))
def test_c_oracle_agrees_with_numpy_restatement_off_defaults(oracle, prm):
    from oracle import tvl1_numpy as N
    kw = dict(BASE, **prm)
    a, b, _ = synth.pair(80, 96, 6)
    fc, lc = oracle.tvl1_calc(a, b, oracle.tvl1_params(**{("lambda" if k == "lambda_" else k): v for k, v in kw.items()}),
                              return_iters=True)
    fn, ln = N.calc(a, b, **{("lam" if k == "lambda_" else k): v for k, v in kw.items()})
    assert np.array_equal(lc, ln), (lc.tolist(), ln.tolist())
    n = len(oracle.tvl1_level_sizes(96, 80, oracle.tvl1_params(nscales=kw["nscales"], scale_step=kw.get("scale_step", 0.8))))
    assert (lc[:n] >= 1).all() and not lc[n:].any()
    if "epsilon" in prm:  # every warp converges at its first check
        assert (lc[:n] == 2).all()
    if "iterations" in prm:
        assert (lc[:n] == prm["iterations"]).all()
    assert np.abs(fc - fn).max() < 5e-4 and synth.aee(fc, fn) < 2e-5
    assert np.isfinite(fc).all()
    assert (np.abs(fc).max() == 0) == (prm.get("lambda_") == 0)  # no data term: u and p stay 0


def _levels(w, h, nscales, step):
    """A.1 restated: round-half-even of the double product (Python's round), stop before a level under 16 pixels"""
    out = [(w, h)]
    while len(out) < nscales:
        nw, nh = round(out[-1][0] * step), round(out[-1][1] * step)
        if nw < 16 or nh < 16:
            break
        out.append((nw, nh))
    return out


def test_level_sizes_off_defaults(oracle):
    sizes = lambda w, h, **kw: oracle.tvl1_level_sizes(w, h, oracle.tvl1_params(**kw))
    # 135 * 0.5 = 67.5 rounds to the even 68
    assert sizes(1920, 1080, nscales=16, scale_step=0.5) == [(1920, 1080), (960, 540), (480, 270), (240, 135), (120, 68), (60, 34), (30, 17)]
    assert sizes(340, 256, nscales=16, scale_step=0.5) == [(340, 256), (170, 128), (85, 64), (42, 32), (21, 16)]
    # 576 * 0.3 = 172.8, 324 * 0.3 = 97.2, 173 * 0.3 = 51.9, 97 * 0.3 = 29.1; then 16 x 9 is dropped
    assert sizes(1920, 1080, nscales=16, scale_step=0.3) == [(1920, 1080), (576, 324), (173, 97), (52, 29)]
    assert sizes(340, 256, nscales=16, scale_step=0.3) == [(340, 256), (102, 77), (31, 23)]
    assert len(sizes(1920, 1080, nscales=16)) == 16 and len(sizes(3840, 2160, nscales=16)) == 16  # the allocated capacity
    assert len(sizes(340, 256, nscales=16)) == 13 and len(sizes(340, 256, nscales=12)) == 12
    assert sizes(1920, 1080, nscales=16)[-1] == (68, 38) and sizes(340, 256, nscales=16)[-1] == (24, 18)  # 340 x 256: 19 x 14 is dropped
    for w, h in ((1920, 1080), (3840, 2160), (340, 256), (131, 97), (96, 80), (17, 16)):
        for step in (0.3, 0.5, 0.7, 0.8, 0.25, 0.75):
            for n in (1, 2, 5, 16):
                assert sizes(w, h, nscales=n, scale_step=step) == _levels(w, h, n, step), (w, h, step, n)


# l_t = lambda * theta and taut = tau / theta of the off-default settings: lambda 0, the default 0.15 at theta 0.05, 1.0 at
# theta 0.3 and at theta 1.0; tau 0.25 at theta 1.0 and at 0.05, tau 1.25 at theta 0.05
L_TS = [np.float32(v) for v in (0.0, 0.15 * 0.05, 0.3, 1.0)]
TAUTS = [np.float32(v) for v in (0.25, 5.0, 25.0)]
THETAS = [np.float32(v) for v in (0.05, 1.0)]
SHAPES = [(16, 16), (37, 53), (131, 97), (1, 8), (13, 13)]


@pytest.mark.parametrize("shape", SHAPES)
def test_primal_and_dual_bounds_off_defaults(oracle, shape):
    w, h = shape
    L = oracle.lib()
    ix, iy, g, rc, u1, u2, p11, p12, p21, p22 = chunk_inputs(w, h, 11 + w)
    for l_t in L_TS:
        for theta in THETAS:
            n1, n2 = u1.copy(), u2.copy()
            err = L.orc_tvl1_estimate_u(ix, iy, g, rc, p11, p12, p21, p22, n1, n2, w, h, l_t, theta, 1)
            ref = r64.primal(ix, iy, g, rc, u1, u2, p11, p12, p21, p22, l_t, theta)
            for name, bad in zip(("u1", "u2"), r64.within_primal(n1, n2, ref)):
                assert not bad.any(), (l_t, theta, name, bad.sum(), tuple(np.argwhere(bad)[0]))
            s, b = r64.convergence_sum(u1, u2, n1, n2, ref)
            assert abs(err - s) <= b, (l_t, theta, err, s, b)
    for taut in TAUTS:
        p = [q.copy() for q in (p11, p12, p21, p22)]
        L.orc_tvl1_estimate_dual(u1, u2, *p, w, h, taut)
        for k, ref in enumerate(r64.dual(u1, u2, p11, p12, p21, p22, taut)):
            _within("taut %g p%d" % (taut, k), p[k], ref)


@pytest.mark.parametrize("step", [0.3, 0.5, 0.7])
def test_upsample_bounds_off_defaults(oracle, step):
    """every level step of 340 x 256 and 131 x 97 at this scale step, times mul = float(1 / scale_step)"""
    mul = np.float32(1.0 / step)
    for w, h in ((340, 256), (131, 97)):
        lv = oracle.tvl1_level_sizes(w, h, oracle.tvl1_params(nscales=16, scale_step=step))
        assert len(lv) >= 2
        for (dw, dh), (sw, sh) in zip(lv, lv[1:]):
            u = (np.random.default_rng(sw * sh).standard_normal((sh, sw)) * 4).astype(np.float32)
            fx, fy = np.float32(1.0 / (dw / sw)), np.float32(1.0 / (dh / sh))
            out = np.empty((dh, dw), np.float32)
            oracle.lib().orc_resize_linear(u, sw, sh, out, dw, dh, fx, fy, 0)
            _within("%dx%d -> %dx%d" % (sw, sh, dw, dh), (out * mul).astype(np.float32), r64.upsample(u, dw, dh, fx, fy, mul))
