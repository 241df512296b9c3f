"""Farneback's Gaussian window (`gaussian_window`) and fast pyramids (`fast_pyramids`; SURVEY B.7) on the GPU.

* Stages: `farn_iteration` on a Gaussian handle (k_box_solve_update<6, true>) and `farn_pyr_down` (k_pyr_down) equal the
  restatement (tests/farn_restate.py) bit for bit in the strict build; in the default build every element is within the
  forward-error bound of tests/farn_ref64.py's float64 restatement.
* Whole flows of the four option combinations through dfb_calc_batch_host: the strict build equals the restatement bit for
  bit, the default build is within AEE 0.01 px of it, at frame sizes from 1 x 200 to 1920 x 1080.
* Batches equal their one-pair calls; every Farneback entry point takes the options; warm starts; a handle switched back
  off gives a fresh handle's bits; a Gaussian handle runs beside a default one; the parameter values taken and refused."""
import threading

import cv2
import numpy as np
import pytest

import farn_cases as fc
import farn_ref64 as r64
import farn_restate as R
from denseflow_b200 import _lib, synth
from oracle import cv_restate

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
COMBOS = [(0, 0), (1, 0), (0, 1), (1, 1)]  # (gaussian_window, fast_pyramids)
AEE_TOL = 0.01  # px, BASELINE.json north_star
_handles = {}


def _new(w, h, variant="strict", **params):
    import denseflow_b200 as d
    e = d.FarnebackOpticalFlow.create(0, w, h, variant)
    for k, v in params.items():
        e.set(k, v)
    return e


def _opts(combo):
    return {"gaussian_window": combo[0], "fast_pyramids": combo[1]}


def _bits_equal(got, want, name):
    diff = got != want
    assert not diff.any(), "%s: %d values differ, first at %s, max |diff| %g" % (
        name, diff.sum(), tuple(np.argwhere(diff)[0]), np.abs(got.astype(np.float64) - want).max())


# ---- stages ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module", autouse=True)
def _module_state():
    """The stage tests' handles and the restated flows live only as long as this module: the handles' device memory (frame
    slots and lanes of a 1080p handle) is returned before later modules create their own large handles."""
    yield
    for e in _handles.values():
        e.release()
    _handles.clear()
    _restated.clear()


def _engine(variant):
    """one 1080p Gaussian handle per build, shared by the stage tests of this module"""
    if variant not in _handles:
        _handles[variant] = _new(1920, 1080, variant, gaussian_window=1)
    return _handles[variant]


ITER_SHAPES = fc.ITER_SHAPES[::3] + fc.ITER_SMALL[::2] + [(1, 1), (13, 13), (340, 256)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("pairs", [1, 3])
def test_gaussian_iteration_stage(oracle, pairs, variant):
    e, orc = _engine(variant), fc.Oracle(oracle)
    for si, (w, h) in enumerate(ITER_SHAPES):
        cases = [orc.pair_case(w, h, 1000 * si + p, fc.FLOW_KINDS[(si + p) % 4]) for p in range(pairs)]
        ins = [fc.stack([c[2][k] for c in cases]) for k in range(5)]
        ins += [fc.stack([c[0][k] for c in cases]) for k in range(5)] + [fc.stack([c[1][k] for c in cases]) for k in range(5)]
        for rebuild in (0, 1):
            out, _ = e.debug_run_kernel("farn_iteration", ins, 7, [rebuild, pairs])
            for p, (R0, R1, M) in enumerate(cases):
                tag = "%dx%d pair %d/%d rebuild %d" % (w, h, p, pairs, rebuild)
                gx, gy = (fc.split(out[i], pairs)[p] for i in (0, 1))
                fx, fy = orc.update_flow(R.gauss_window5(M))
                rx, ry, rM = (r64.gauss_iteration(M, R0, R1, gx, gy, R.gauss_weights()) if variant == "default"
                              else (None, None, [None] * 5))
                fc.check(variant, tag + " fx", gx, fx, rx)
                fc.check(variant, tag + " fy", gy, fy, ry)
                if rebuild:
                    Mp = orc.update_matrices(fx, fy, R0, R1) if variant == "strict" else [None] * 5
                    for k in range(5):
                        fc.check(variant, "%s M'%d" % (tag, k), fc.split(out[2 + k], pairs)[p], Mp[k], rM[k])


@pytest.mark.parametrize("variant", VARIANTS)
def test_pyr_down_stage(variant):
    e = _engine(variant)
    for w, h in fc.FRAME_SHAPES + fc.SMALL_FRAMES + [(45, 90), (43, 32), (85, 64)]:
        img = fc.frame_f32(w, h, 5)
        img[::3] -= 128.0  # signed values too
        (got,), _ = e.debug_run_kernel("farn_pyr_down", [img], 1, out_shape=((h + 1) // 2, (w + 1) // 2))
        fc.check(variant, "%dx%d pyrDown" % (w, h), got, R.pyr_down(img), None if variant == "strict" else r64.pyr_down(img))


# ---- whole flows -------------------------------------------------------------------------------------------------------------
FLOW_SHAPES = [(256, 256), (256, 340), (256, 455), (720, 1280), (49, 33), (7, 5), (200, 1), (1080, 1920)]
_restated = {}


def _restatement(a, b, key, combo, init=None, params=None):
    k = (key, combo, init is not None)
    if k not in _restated:
        _restated[k] = R.farn_calc(a, b, init=init, params=params, **_opts(combo))
    return _restated[k]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("combo", COMBOS)
@pytest.mark.parametrize("shape", FLOW_SHAPES)
def test_whole_flow(oracle, shape, combo, variant):
    h, w = shape
    a, b, _ = synth.pair(h, w, 7)
    e = _new(w, h, variant, **_opts(combo))
    got = e.calc_batch([a, b], step=1)[0]
    want = _restatement(a, b, shape, combo)
    if variant == "strict":
        _bits_equal(got, want, "%dx%d %s" % (w, h, combo))
    else:
        aee = float(np.hypot(*(got.astype(np.float64) - want).transpose(2, 0, 1)).mean())
        assert aee <= AEE_TOL, (shape, combo, aee)
    e.release()


def test_options_change_the_flow():
    h, w = 256, 340
    a, b, _ = synth.pair(h, w, 7)
    flows = [_new(w, h, "default", **_opts(c)).calc(a, b) for c in COMBOS]
    for i in range(4):
        for j in range(i):
            assert (flows[i] != flows[j]).any(), (COMBOS[i], COMBOS[j])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("combo", COMBOS[1:])
def test_batches_equal_single_pairs(variant, combo):
    import torch
    h, w = 97, 131
    fr = synth.stream(h, w, 12, seed=11)
    e = _new(w, h, variant, **_opts(combo))
    dfr = torch.from_numpy(np.ascontiguousarray(fr)).cuda()
    for step in (1, -3):
        host = e.calc_batch(list(fr), step=step)
        dev = e.calc_batch_device(dfr, step=step).cpu().numpy()
        for j in range(host.shape[0]):
            a, b = (fr[j], fr[j + step]) if step > 0 else (fr[j - step], fr[j])
            one = e.calc(a, b)
            _bits_equal(host[j], one, "step %d pair %d host batch" % (step, j))
            _bits_equal(dev[j], one, "step %d pair %d device batch" % (step, j))
            _bits_equal(e.calc(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()).cpu().numpy(), one, "calc_device pair %d" % j)
    e.release()


@pytest.mark.parametrize("combo", COMBOS[1:])
def test_every_entry_point_takes_the_options(oracle, combo):
    """the float, planar, quantised (the CAST quantisation of the float flow), PNG and colour-chain calls agree with calc_batch"""
    import torch
    import denseflow_b200 as d
    h, w, bound = 96, 128, 20
    gray = synth.stream(h, w, 6, seed=5)
    bgr = np.stack([np.stack([f, np.roll(f, 3, 1), 255 - f], -1) for f in gray])
    e = d.create("farn", 0, w, h)
    for k, v in _opts(combo).items():
        e.set(k, v)
    flows = e.calc_batch(list(gray), step=1)
    _bits_equal(e.calc_batch_planes(list(gray), step=1), flows.transpose(0, 3, 1, 2), "calc_batch_planes")
    dev = torch.from_numpy(np.ascontiguousarray(gray)).cuda()
    _bits_equal(e.calc_batch_device_planes(dev, step=1).cpu().numpy(), flows.transpose(0, 3, 1, 2), "calc_batch_device_planes")
    qx, qy = e.calc_batch(list(gray), step=1, bound=bound)
    for j in range(flows.shape[0]):
        rx, ry = oracle.quantise(flows[j], bound)
        assert np.array_equal(qx[j], rx) and np.array_equal(qy[j], ry), j
    for i, png in enumerate(e.calc_batch_png(list(gray), step=1)):
        img = cv2.imdecode(np.frombuffer(bytes(png), np.uint8), cv2.IMREAD_COLOR)
        assert np.array_equal(img, cv_restate.flow_to_png_image(flows[i])[0]), i
    g2 = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]
    _bits_equal(e.process_bgr_batch_planes(bgr, step=1), e.calc_batch(g2, step=1).transpose(0, 3, 1, 2), "process_bgr_batch_planes")
    e.release()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("combo", COMBOS[1:])
@pytest.mark.parametrize("shape,levels", [((97, 131), 5), ((256, 340), 5), ((256, 340), 0)])
def test_warm_start(oracle, shape, levels, combo, variant):
    h, w = shape
    a, b, _ = synth.pair(h, w, 9)
    init = np.ascontiguousarray(R.farn_calc(a, b) * np.float32(0.6) + np.float32(0.25))
    e = _new(w, h, variant, num_levels=levels, use_initial_flow=1, **_opts(combo))
    got = e.calc(a, b, flow=init.copy())
    want = R.farn_calc(a, b, init=init, params=oracle.farn_params(num_levels=levels), **_opts(combo))
    if variant == "strict":
        _bits_equal(got, want, "%dx%d levels %d %s" % (w, h, levels, combo))
    else:
        assert float(np.hypot(*(got.astype(np.float64) - want).transpose(2, 0, 1)).mean()) <= AEE_TOL
    cold = R.farn_calc(a, b, params=oracle.farn_params(num_levels=levels), **_opts(combo))
    assert (want != cold).any()
    e.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_switched_off_again_equals_a_fresh_handle(variant):
    h, w = 256, 340
    fr = synth.stream(h, w, 4, seed=3)
    fresh = _new(w, h, variant)
    want = fresh.calc_batch(list(fr), step=1)
    fresh.release()
    e = _new(w, h, variant)
    for combo in COMBOS[1:]:
        for k, v in _opts(combo).items():
            e.set(k, v)
        assert (e.calc_batch(list(fr), step=1) != want).any(), combo
        e.set("gaussian_window", 0).set("fast_pyramids", 0)
        _bits_equal(e.calc_batch(list(fr), step=1), want, "%s switched off" % (combo,))
    e.release()


def test_gaussian_handle_beside_default_handle():
    h, w = 256, 340
    fr = synth.stream(h, w, 6, seed=6)
    plain = _new(w, h, "default")
    want = plain.calc_batch(list(fr), step=1)
    gau = _new(w, h, "default", gaussian_window=1, fast_pyramids=1)
    alone = gau.calc_batch(list(fr), step=1)
    got, errors = {}, []

    def run():
        try:
            for i in range(2):
                got[i] = gau.calc_batch(list(fr), step=1)
        except Exception as ex:  # surfaced below
            errors.append(ex)

    t = threading.Thread(target=run)
    t.start()
    plain_runs = [plain.calc_batch(list(fr), step=1) for _ in range(2)]
    t.join()
    assert not errors, errors
    for i, f in enumerate(plain_runs):
        _bits_equal(f, want, "default handle, run %d beside the Gaussian handle" % i)
    for i in range(2):
        _bits_equal(got[i], alone, "Gaussian handle, run %d beside the default handle" % i)
    plain.release()
    gau.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_parameter_table(variant):
    import denseflow_b200 as d
    e = _new(64, 64, variant)
    L = _lib.load(variant)
    for name in ("gaussian_window", "fast_pyramids"):
        assert e.get(name) == 0
        for v in (1, 0, 1):
            e.set(name, v)
            assert e.get(name) == v
        for v in (2, 0.5, -1, 1e9, float("nan"), float("inf"), float("-inf")):
            assert L.dfb_set_param(e._h, name.encode(), float(v)) == _lib.DFB_ERR_INVALID_ARG, (name, v)
            assert L.dfb_last_error(e._h).decode() == "bad parameter " + name, (name, v)
            assert e.get(name) == 1, (name, v)
    e.release()
    t = d.OpticalFlowDual_TVL1.create(0, 64, 64, variant)
    for name in ("gaussian_window", "fast_pyramids"):
        assert L.dfb_set_param(t._h, name.encode(), 0.0) == _lib.DFB_ERR_INVALID_ARG
        assert L.dfb_last_error(t._h).decode() == "bad parameter " + name
    t.release()
