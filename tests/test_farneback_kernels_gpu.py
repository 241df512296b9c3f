"""Per-stage parity of the Farneback kernels, launched through the engine's own launch code (dfb_debug_run_kernel "farn_*"
stages), and end-to-end pins of the whole flow.

* strict build (IEEE, no FMA contraction, correctly rounded division): it performs the oracle's fp32 operations in the
  oracle's order, so every stage and every flow must EQUAL the oracle's building block / orc_farn_calc bit for bit;
* default build: every element within the forward-error bound of the float64 restatement (tests/farn_ref64.py), element
  by element."""
import numpy as np
import pytest

import farn_cases as fc
import farn_ref64 as r64
from denseflow_b200 import synth

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
_handles = {}


def _engine(variant):
    """one 1080p handle per build, shared by the stage tests (the hook writes into its frame slots and lanes)"""
    if variant not in _handles:
        import denseflow_b200 as d
        _handles[variant] = d.FarnebackOpticalFlow.create(0, 1920, 1080, variant)
    return _handles[variant]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("shape", fc.FRAME_SHAPES + fc.SMALL_FRAMES)
def test_level_image_and_poly_exp(oracle, shape, variant):
    """k_gauss_blur (k = 0), k_gauss_vert_rows + k_gauss_horz_resize (k > 0) and k_poly_exp<5> at every level"""
    w, h = shape
    e, orc = _engine(variant), fc.Oracle(oracle)
    frame = fc.frame_f32(w, h, 3)
    for k in range(len(oracle.farn_levels(w, h))):
        want, (lw, lh, smooth, sigma) = orc.level_image(frame, k)
        (img,), _ = e.debug_run_kernel("farn_level_image", [frame], 1, [k], out_shape=(lh, lw))
        fc.check(variant, "%dx%d level %d image" % (w, h, k), img, want, None if variant == "strict" else r64.level_image(frame, lw, lh, smooth, sigma))
        R, _ = e.debug_run_kernel("farn_poly_exp", [want], 5)
        Rw = orc.poly_exp(want)
        refs = r64.poly_exp(want) if variant == "default" else [None] * 5
        for i in range(5):
            fc.check(variant, "%dx%d level %d R%d" % (w, h, k, i), R[i], Rw[i], refs[i])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("w", fc.ITER_W + fc.SMALL_W)
def test_update_matrices(oracle, w, variant):
    """k_update_matrices: the four flow kinds as four pairs of one launch, every iteration height (every small height for
    the widths below 32)"""
    e, orc = _engine(variant), fc.Oracle(oracle)
    for h in (fc.ITER_H if w >= 32 else fc.SMALL_H):
        cases = []
        for p, kind in enumerate(fc.FLOW_KINDS):
            R0, R1 = orc.expansions(w, h, 100 + p)
            cases.append((kind, fc.flow(kind, w, h, w * 7 + h + p), R0, R1))
        ins = [fc.stack([c[1][0] for c in cases]), fc.stack([c[1][1] for c in cases])]
        ins += [fc.stack([c[2][k] for c in cases]) for k in range(5)] + [fc.stack([c[3][k] for c in cases]) for k in range(5)]
        M, _ = e.debug_run_kernel("farn_update_matrices", ins, 5, [len(cases)])
        for p, (kind, (fx, fy), R0, R1) in enumerate(cases):
            want = orc.update_matrices(fx, fy, R0, R1)
            refs = r64.update_matrices(fx, fy, R0, R1) if variant == "default" else [None] * 5
            for k in range(5):
                fc.check(variant, "%dx%d %s M%d" % (w, h, kind, k), fc.split(M[k], len(cases))[p], want[k], refs[k])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("pairs", [1, 3, 8])
def test_iteration(oracle, pairs, variant):
    """k_box_solve_update<6>: every iteration shape, with and without the rebuild of M, several
    pairs with different data in one launch (the persistent kernel's tile list runs over pairs x tile rows x tile columns)"""
    e, orc = _engine(variant), fc.Oracle(oracle)
    for si, (w, h) in enumerate(fc.ITER_SHAPES + fc.ITER_SMALL):
        cases = [orc.pair_case(w, h, 1000 * si + p, fc.FLOW_KINDS[(si + p) % 4]) for p in range(pairs)]
        ins = [fc.stack([c[2][k] for c in cases]) for k in range(5)]
        ins += [fc.stack([c[0][k] for c in cases]) for k in range(5)] + [fc.stack([c[1][k] for c in cases]) for k in range(5)]
        for rebuild in (0, 1):
            out, _ = e.debug_run_kernel("farn_iteration", ins, 7, [rebuild, pairs])
            for p, (R0, R1, M) in enumerate(cases):
                tag = "%dx%d pair %d/%d rebuild %d" % (w, h, p, pairs, rebuild)
                gx, gy = (fc.split(out[i], pairs)[p] for i in (0, 1))
                fx, fy, Mp = orc.iteration(M, R0, R1, rebuild)
                rx, ry, rM = r64.iteration(M, R0, R1, gx, gy) if variant == "default" else (None, None, [None] * 5)
                fc.check(variant, tag + " fx", gx, fx, rx)
                fc.check(variant, tag + " fy", gy, fy, ry)
                if rebuild:
                    for k in range(5):
                        fc.check(variant, "%s M'%d" % (tag, k), fc.split(out[2 + k], pairs)[p], Mp[k], rM[k])


@pytest.mark.parametrize("variant", VARIANTS)
def test_flow_init(oracle, variant):
    """k_flow_init: the level-start upsample x 2 between every two consecutive levels of the frame shapes"""
    e, orc = _engine(variant), fc.Oracle(oracle)
    for w, h in fc.FRAME_SHAPES:
        lv = oracle.farn_levels(w, h)
        for i in range(1, len(lv)):
            (pw, ph), (lw, lh) = lv[i - 1][:2], lv[i][:2]
            pfx, pfy = fc.flow("smooth", pw, ph, i)
            pfx[::7] = fc.flow("iid", pw, ph, i)[0][::7]
            got, _ = e.debug_run_kernel("farn_flow_init", [pfx, pfy], 2, [lw, lh], out_shape=(lh, lw))
            want = orc.flow_init(pfx, pfy, lw, lh)
            refs = r64.flow_init(pfx, pfy, lw, lh) if variant == "default" else [None, None]
            for c in range(2):
                fc.check(variant, "%dx%d -> %dx%d flow %d" % (pw, ph, lw, lh, c), got[c], want[c], refs[c])


# ---- end to end ---------------------------------------------------------------------------------------------------------

def _new(w, h, variant="strict"):
    import denseflow_b200 as d
    return d.FarnebackOpticalFlow.create(0, w, h, variant)


def _assert_equal(got, want, name):
    diff = np.any(got != want, axis=-1) if got.ndim == 3 else got != want
    assert not diff.any(), "%s: %d pixels differ, first at %s, max |diff| %g" % (
        name, diff.sum(), tuple(np.argwhere(diff)[0]), np.abs(got.astype(np.float64) - want).max())


@pytest.mark.parametrize("shape", [(256, 256), (256, 340), (97, 131), (64, 64), (360, 640)])
def test_strict_flow_is_bit_exact(oracle, shape):
    h, w = shape
    a, b, _ = synth.pair(h, w, 0)
    e = _new(w, h)
    _assert_equal(e.calc(a, b), oracle.farn_calc(a, b), "%dx%d" % (w, h))


@pytest.mark.parametrize("params", [{"num_levels": 0}, {"num_levels": 1}, {"num_levels": 3}, {"num_iters": 1},
                                    {"num_iters": 2}, {"poly_sigma": 1.5}, {"num_levels": 3, "num_iters": 1}])
def test_strict_flow_is_bit_exact_under_parameter_changes(oracle, params):
    """num_levels 5 / num_iters 10 are the defaults above; num_iters = 1 runs only the iteration without rebuild"""
    h, w = 97, 131
    a, b, _ = synth.pair(h, w, 4)
    e = _new(w, h)
    for k, v in params.items():
        e.set(k, v)
    _assert_equal(e.calc(a, b), oracle.farn_calc(a, b, oracle.farn_params(**params)), str(params))


def test_default_flow_regression_guard(oracle):
    """Tighter than the 0.01 px contract of test_farneback_matches_oracle: overall AEE, AEE of the 6-pixel border band (the
    reach of c_border and of the box half-width) and the 99.9th percentile of the per-pixel EPE against the oracle.
    Measured on an H100 80 GB (default build) at 640 x 360: AEE 5.75e-07, border-band AEE 6.92e-07, p99.9 EPE 4.64e-06 px;
    the guards are ~10x those."""
    h, w = 360, 640
    a, b, _ = synth.pair(h, w, 0)
    flow = _new(w, h, "default").calc(a, b)
    ref = oracle.farn_calc(a, b)
    epe = np.hypot(*(flow.astype(np.float64) - ref).transpose(2, 0, 1))
    band = np.ones((h, w), bool)
    band[6:-6, 6:-6] = False
    aee, aee_band, p999 = epe.mean(), epe[band].mean(), np.percentile(epe, 99.9)
    print("default build vs oracle: AEE %.3g, border-band AEE %.3g, p99.9 EPE %.3g px" % (aee, aee_band, p999))
    assert aee <= 6e-6 and aee_band <= 7e-6 and p999 <= 5e-5


@pytest.mark.parametrize("variant", VARIANTS)
def test_long_batches_equal_single_pairs(oracle, variant):
    """20 frames at step 1 (three solve groups, 8 + 8 + 3 pairs, frame slots reused around the ring) and at step +-9 (a
    larger ring and look-ahead): every flow equals the single-pair calc of its frames, and the oracle in the strict build"""
    h, w = 97, 131
    fr = synth.stream(h, w, 20, seed=8)
    e = _new(w, h, variant)
    for step in (1, 9, -9):
        flows = e.calc_batch(list(fr), step=step)
        assert flows.shape[0] == 20 - abs(step)
        for j in range(flows.shape[0]):
            a, b = (fr[j], fr[j + step]) if step > 0 else (fr[j - step], fr[j])
            _assert_equal(flows[j], e.calc(a, b), "step %d pair %d vs calc" % (step, j))
            if variant == "strict" and (j % 4 == 0 or j == flows.shape[0] - 1):
                _assert_equal(flows[j], oracle.farn_calc(a, b), "step %d pair %d vs oracle" % (step, j))


@pytest.mark.parametrize("variant", VARIANTS)
def test_one_handle_many_sizes(oracle, variant):
    """one handle serves several frame sizes and parameter changes back to back (the tensor-map cache key, the slot layout of
    smaller frames): every flow equals a fresh handle's (and the oracle's in the strict build)"""
    e = _new(640, 360, variant)
    runs = [((360, 640), {}), ((97, 131), {}), ((64, 64), {"num_iters": 3}), ((201, 333), {"num_levels": 3, "num_iters": 10}),
            ((360, 640), {}), ((97, 131), {"num_levels": 5}), ((256, 340), {"num_iters": 10})]
    for i, ((h, w), params) in enumerate(runs):
        for k, v in params.items():
            e.set(k, v)
        cur = {k: e.get(k) for k in ("num_levels", "num_iters")}
        a, b, _ = synth.pair(h, w, 20 + i)
        got = e.calc(a, b)
        fresh = _new(w, h, variant)
        for k, v in cur.items():
            fresh.set(k, v)
        _assert_equal(got, fresh.calc(a, b), "run %d %dx%d vs fresh handle" % (i, w, h))
        if variant == "strict":
            op = oracle.farn_params(num_levels=int(cur["num_levels"]), num_iters=int(cur["num_iters"]))
            _assert_equal(got, oracle.farn_calc(a, b, op), "run %d %dx%d vs oracle" % (i, w, h))
