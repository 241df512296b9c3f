"""The oracle's Farneback building blocks, one at a time, against the float64 restatement of tests/farn_ref64.py: every
fp32 output element must lie within the forward-error bound derived for its operation.  This keeps those bounds honest
without a GPU (tests/test_farneback_kernels_gpu.py holds the default build's kernels to the same bounds)."""
import numpy as np
import pytest

import farn_cases as fc
import farn_ref64 as r64


def _within(name, got, ref):
    """fc.within, and every bound finite: a bound of inf would pass anything"""
    fc.within(name, got, ref)
    assert np.isfinite(ref[1]).all()


def test_levels_and_constants_match_the_oracle(oracle):
    for w, h in fc.FRAME_SHAPES + [(160, 96), (64, 64)]:
        for nl in (0, 1, 3, 5):
            want = oracle.farn_levels(w, h, oracle.farn_params(num_levels=nl))
            got = r64.levels(w, h, nl)
            assert [g[:3] for g in got] == [x[:3] for x in want] and np.allclose([g[3] for g in got], [x[3] for x in want])
    g, xg, xxg, ig = (np.empty(6, np.float32), np.empty(6, np.float32), np.empty(6, np.float32), np.empty(4, np.float32))
    oracle.lib().orc_farn_poly_constants(5, 1.1, g, xg, xxg, ig)
    mine = r64.poly_constants(5, 1.1)
    for a, b in zip((g, xg, xxg, ig), mine):  # within the one rounding the reference allows for constants
        assert np.all(np.abs(a.astype(np.float64) - b) <= 2 ** -24 * np.abs(b) * 1.0000001)


@pytest.mark.parametrize("shape", fc.FRAME_SHAPES + fc.SMALL_FRAMES)
def test_level_image_and_poly_exp_within_bounds(oracle, shape):
    w, h = shape
    orc = fc.Oracle(oracle)
    frame = fc.frame_f32(w, h, 3)
    for k in range(len(r64.levels(w, h))):
        img, (lw, lh, smooth, sigma) = orc.level_image(frame, k)
        assert img.shape == (lh, lw)
        _within("level %d image" % k, img, r64.level_image(frame, lw, lh, smooth, sigma))
        if lw * lh <= 640 * 360:  # the polynomial expansion at full HD is covered by the smaller frames' levels
            R = orc.poly_exp(img)
            for i, ref in enumerate(r64.poly_exp(img)):
                _within("level %d R%d" % (k, i), R[i], ref)


@pytest.mark.parametrize("shape", [(32, 32), (33, 49), (47, 37), (97, 38), (340, 256), (1, 1), (2, 1), (1, 3), (3, 2), (5, 7), (8, 8),
                                   (12, 5), (13, 13), (17, 31), (1, 200), (200, 2)])
def test_pair_stages_within_bounds(oracle, shape):
    w, h = shape
    orc = fc.Oracle(oracle)
    R0, R1 = orc.expansions(w, h, 5)
    for kind in fc.FLOW_KINDS:
        fx, fy = fc.flow(kind, w, h, 11)
        M = orc.update_matrices(fx, fy, R0, R1)
        for i, ref in enumerate(r64.update_matrices(fx, fy, R0, R1)):
            _within("%s M%d" % (kind, i), M[i], ref)
        B = orc.box_filter5(M)
        for i, ref in enumerate(r64.box_mean(M)):
            _within("%s box mean %d" % (kind, i), B[i], ref.out())
        gx, gy = orc.update_flow(B)
        rx, ry = r64.update_flow(B)
        _within(kind + " solve x", gx, rx)
        _within(kind + " solve y", gy, ry)
        # the whole iteration from M, as the fused kernel computes it
        ix, iy, Mp = r64.iteration(M, R0, R1, gx, gy)
        _within(kind + " iteration x", gx, ix)
        _within(kind + " iteration y", gy, iy)
        Mo = orc.update_matrices(gx, gy, R0, R1)
        for i, ref in enumerate(Mp):
            _within("%s rebuilt M%d" % (kind, i), Mo[i], ref)
        lw, lh = 2 * w - 1, 2 * h + 1  # odd sizes: the clamp of the far tap binds
        for got, ref in zip(orc.flow_init(fx, fy, lw, lh), r64.flow_init(fx, fy, lw, lh)):
            _within(kind + " flow init", got, ref)


def test_bounds_are_tight_enough_to_see_a_one_column_shift(oracle):
    """A bound is only useful if it is much smaller than the errors the kernels are prone to: moving the right c_border
    band by one column (the weight 0.4472 instead of 1) must fall far outside it."""
    w, h = 47, 37
    orc = fc.Oracle(oracle)
    R0, R1 = orc.expansions(w, h, 5)
    fx, fy = fc.flow("smooth", w, h, 3)
    M = orc.update_matrices(fx, fy, R0, R1)
    wrong = M[:, :, w - 6] * np.float32(0.4472 ** 2)  # x = w - 6: min(w - x - 1, 5) = 5, shifted: 4
    v, b = r64.update_matrices(fx, fy, R0, R1)[0]
    assert (np.abs(wrong[0] - v[:, w - 6]) > 100 * b[:, w - 6]).mean() > 0.9
