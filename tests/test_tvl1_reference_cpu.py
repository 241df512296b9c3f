"""The oracle's TV-L1 building blocks, one at a time, against the float64 restatement of tests/tvl1_ref64.py: every fp32
output element must lie within the forward-error bound derived for its operation.  This keeps those bounds honest without
a GPU (tests/test_tvl1_kernels_gpu.py and tests/test_tvl1_fused_stages_gpu.py hold the default build to the same bounds).
Also: the oracle's flow does not depend on its thread count (the convergence sum is reduced in a thread-dependent order)."""
import numpy as np
import pytest

import tvl1_ref64 as r64
from denseflow_b200 import synth
from tvl1_cases import chunk_inputs, warp_flow

L_T, TAUT, THETA = np.float32(0.15 * 0.3), np.float32(0.25 / 0.3), np.float32(0.3)
SHAPES = [(16, 16), (37, 53), (131, 97), (340, 256)]
# below the level cut (tests/geometry_cases.py): single pixels, rows, columns, one four-pixel group, thin strips
SMALL = [(1, 1), (2, 1), (1, 2), (3, 2), (2, 3), (4, 4), (1, 8), (8, 1), (5, 7), (13, 13), (15, 12), (1, 400), (400, 1), (7, 300)]


def _within(name, got, ref):
    v, b = ref
    bad = ~(np.abs(got.astype(np.float64) - v) <= b)
    assert not bad.any(), "%s: %d elements outside the bound, first at %s: got %r, float64 %r, bound %r" % (
        name, bad.sum(), tuple(np.argwhere(bad)[0]), got[bad][0], v[bad][0], b[bad][0])
    assert np.isfinite(b).all()


@pytest.mark.parametrize("shape", SHAPES + SMALL)
def test_gradient_and_warp_within_bounds(oracle, shape):
    w, h = shape
    L = oracle.lib()
    rng = np.random.default_rng(w + h)
    I0 = np.rint(rng.random((h, w)) * 255).astype(np.float32)
    I1 = np.rint(rng.random((h, w)) * 255).astype(np.float32)
    gx, gy = np.empty_like(I1), np.empty_like(I1)
    L.orc_centered_gradient(I1, w, h, gx, gy)
    rx, ry = r64.gradient(I1)
    _within("I1x", gx, rx)
    _within("I1y", gy, ry)
    u1, u2 = warp_flow(w, h, 3)
    outs = [np.empty_like(I1) for _ in range(5)]
    L.orc_tvl1_warp_backward(I0, I1, gx, gy, u1, u2, w, h, *outs)
    for got, ref, name in zip(outs[1:], r64.warp(I0, I1, gx, gy, u1, u2), ["I1wx", "I1wy", "grad", "rho_c"]):
        _within(name, got, ref)


@pytest.mark.parametrize("shape", SHAPES + SMALL)
def test_primal_dual_and_error_within_bounds(oracle, shape):
    w, h = shape
    L = oracle.lib()
    ix, iy, g, rc, u1, u2, p11, p12, p21, p22 = chunk_inputs(w, h, 7)
    n1, n2 = u1.copy(), u2.copy()
    err = L.orc_tvl1_estimate_u(ix, iy, g, rc, p11, p12, p21, p22, n1, n2, w, h, L_T, THETA, 1)
    ref = r64.primal(ix, iy, g, rc, u1, u2, p11, p12, p21, p22, L_T, THETA)
    for name, bad in zip(("u1", "u2"), r64.within_primal(n1, n2, ref)):
        assert not bad.any(), (name, bad.sum(), tuple(np.argwhere(bad)[0]))
    assert ref[3].any()  # the g <= FLT_EPSILON exception is exercised
    s, b = r64.convergence_sum(u1, u2, n1, n2, ref)
    assert abs(err - s) <= b, (err, s, b)
    p = [q.copy() for q in (p11, p12, p21, p22)]
    L.orc_tvl1_estimate_dual(n1, n2, *p, w, h, TAUT)
    for k, ref in enumerate(r64.dual(n1, n2, p11, p12, p21, p22, TAUT)):
        _within("p%d" % k, p[k], ref)


@pytest.mark.parametrize("src, dst", [((54, 40), (67, 50)), ((105, 78), (131, 97)), ((272, 205), (340, 256)), ((1, 1), (1, 1)),
                                      ((1, 1), (5, 3)), ((2, 1), (3, 1)), ((1, 6), (1, 8)), ((10, 10), (13, 13)), ((320, 1), (400, 1))])
def test_upsample_within_bounds(oracle, src, dst):
    (sw, sh), (dw, dh) = src, dst
    u = (np.random.default_rng(sw).standard_normal((sh, sw)) * 4).astype(np.float32)
    fx, fy = np.float32(1.0 / (dw / sw)), np.float32(1.0 / (dh / sh))
    out = np.empty((dh, dw), np.float32)
    oracle.lib().orc_resize_linear(u, sw, sh, out, dw, dh, fx, fy, 0)
    out = (out * np.float32(1.0 / 0.8)).astype(np.float32)
    _within("upsample", out, r64.upsample(u, dw, dh, fx, fy, 1.0 / 0.8))


def test_bounds_are_tight_enough_to_see_a_missing_mirror(oracle):
    """A dual step that forgets the index clamp at the last column (u(W) taken as 0 instead of u(W - 1)) must fall far outside
    the bound there: the bounds are a few ulps, not a tolerance."""
    w, h = 37, 53
    _, _, _, _, u1, u2, p11, p12, p21, p22 = chunk_inputs(w, h, 9)
    pad = lambda u: np.ascontiguousarray(np.concatenate([u, np.zeros((h, 1), np.float32)], axis=1))
    wrong = [pad(q) for q in (p11, p12, p21, p22)]
    oracle.lib().orc_tvl1_estimate_dual(pad(u1), pad(u2), *wrong, w + 1, h, TAUT)
    v, b = r64.dual(u1, u2, p11, p12, p21, p22, TAUT)[0]
    assert (np.abs(wrong[0][:, w - 1] - v[:, w - 1]) > 100 * b[:, w - 1]).mean() > 0.9


@pytest.mark.parametrize("shape", [(97, 131), (256, 256)])
def test_oracle_flow_is_independent_of_its_thread_count(oracle, shape):
    h, w = shape
    a, b, _ = synth.pair(h, w, 0)
    L = oracle.lib()
    try:
        L.orc_set_num_threads(1)
        one, log1, errs1 = oracle.tvl1_calc(a, b, return_iters=True, return_errors=True)
        L.orc_set_num_threads(8)
        eight, log8, errs8 = oracle.tvl1_calc(a, b, return_iters=True, return_errors=True)
    finally:
        L.orc_set_num_threads(min(8, oracle.usable_cores()))
    assert np.array_equal(one, eight) and np.array_equal(log1, log8)
    assert len(errs1) == len(errs8) and np.allclose(errs1[:, 0], errs8[:, 0], rtol=1e-12, atol=0)


def test_geometry_cases_count_levels_as_the_oracles_do(oracle):
    """tests/geometry_cases.py restates both pyramid rules to place its level cuts: they must agree with the oracles'"""
    import geometry_cases as gc
    shapes = gc.TINY + gc.SQUARES + gc.STRIPS + gc.LARGE + gc.TVL1_CUTS + gc.FARN_CUTS + gc.STAGE_SMALL + gc.STAGE_STRIPS
    for w, h in shapes:
        assert gc.tvl1_levels(w, h) == len(oracle.tvl1_level_sizes(w, h)), (w, h)
        assert gc.farn_levels(w, h) == len(oracle.farn_levels(w, h)), (w, h)
    for cuts, levels in ((gc.TVL1_CUTS, gc.tvl1_levels), (gc.FARN_CUTS, gc.farn_levels)):
        assert all(levels(*cuts[i]) + 1 == levels(*cuts[i + 1]) for i in range(0, len(cuts), 2))
