"""The TV-L1 illumination term (`gamma`; SURVEY.md A.8, DESIGN §4.3) on the GPU.

* Stages: the gamma primal and dual kernels (the `estimate_u_gamma` / `estimate_dual_gamma` stages of dfb_debug_run_kernel)
  equal the restatement's steps (tests/tvl1_restate.py) bit for bit in the strict build, on frame-sized, tiny and thin
  planes, convergence sum included.
* Strict build: flows and per-(scale, warp) iteration logs equal the restatement over the C oracle's building blocks bit for
  bit, in both schedules (the fused gamma kernel k_tvl1_pair_gamma and the per-half-step kernels), on 256 x 256, the tiny and
  thin shapes, a fade, pairs of a 340 x 256 clip at 1 / 3 / automatic lanes, with the median and with a warm start.
* Both builds: the fused gamma kernel equals the per-half-step schedule bit for bit (flows and logs) on a 63-pair 340 x 256
  clip and a 1920 x 1080 batch at 1 / 3 / automatic lanes, with the median and with warm starts.  fused_k and use_tma
  configure the tile loop, which the gamma kernel does not run: they must not change its bits either.
* Default build: within 0.01 px of the restatement; batches equal per-pair calls; every flow entry point gives bytes
  consistent with calc_batch; gamma set back to 0 gives a fresh handle's bits; a gamma handle beside a default handle on one
  GPU gives each its own result.
* Parameter: finite values >= 0 are taken, NaN, +-inf and negative values refused with the old value kept; Farneback handles
  refuse the name."""
import threading

import cv2
import numpy as np
import pytest

import content_cases as cc
import geometry_cases as gc
import tvl1_pin as pin
import tvl1_restate as T
from denseflow_b200 import _lib, synth
from oracle import cv_restate

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
AEE_TOL = 0.01  # px, BASELINE.json north_star


def _new(w, h, variant="strict", **params):
    import denseflow_b200 as d
    e = d.OpticalFlowDual_TVL1.create(0, w, h, variant)
    for k, v in params.items():
        e.set(k, v)
    return e


def _bits_equal(got, want, what):
    bad = np.asarray(got).view(np.int32) != np.asarray(want).view(np.int32)
    assert not bad.any(), "%s: %d of %d differ, first at %s" % (what, bad.sum(), bad.size, tuple(np.argwhere(bad)[0]))


def _brighter(b, gain=1.1, offset=8.0):
    return np.clip(np.rint(b.astype(np.float64) * gain + offset), 0, 255).astype(np.uint8)


ORACLE_KEYS = ("nscales", "warps", "iterations", "epsilon", "tau", "theta", "lambda", "scale_step")


def _reference(a, b, gamma, params, init=None):
    op = {n: v for n, v in params.items() if n in ORACLE_KEYS}
    med = {n: v for n, v in params.items() if n.startswith("median_")}
    return T.tvl1_calc(a, b, gamma=gamma, init=init, **med, **op)


# ---- stages --------------------------------------------------------------------------------------------------------------
def _stage_inputs(w, h, seed):
    rng = np.random.default_rng(seed)
    ix = (rng.standard_normal((h, w)) * 8).astype(np.float32)
    iy = (rng.standard_normal((h, w)) * 8).astype(np.float32)
    ix[::5, ::3] = 0
    iy[::5, ::3] = 0  # grad <= eps
    grad = (ix * ix + iy * iy).astype(np.float32)
    rho_c = (rng.standard_normal((h, w)) * 20).astype(np.float32)
    p = [rng.uniform(-1, 1, (h, w)).astype(np.float32) for _ in range(6)]
    u = [rng.standard_normal((h, w)).astype(np.float32) for _ in range(3)]
    return ix, iy, grad, rho_c, p, u


STAGE_SHAPES = [(37, 53), (128, 131), (480, 270)] + gc.TINY[::5] + gc.STAGE_STRIPS


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("gamma", [0.1, 1.0, 7.5])
def test_stages_equal_the_restatement(variant, gamma):
    e = _new(64, 64, variant)
    l_t, theta, taut = np.float32(0.15 * 0.3), np.float32(0.3), np.float32(0.25 / 0.3)
    for j, (w, h) in enumerate(STAGE_SHAPES):
        ix, iy, grad, rho_c, p, u = _stage_inputs(w, h, 100 * j + int(gamma * 10))
        r1, r2, r3, err_ref = T.estimate_u_gamma(ix, iy, grad, rho_c, *p, *u, l_t, theta, gamma)
        (g1, g2, g3), err = e.debug_run_kernel("estimate_u_gamma", [ix, iy, grad, rho_c, *p, *u], 3,
                                               [float(l_t), float(theta), 1, gamma])
        pr = [q.copy() for q in p]
        T.estimate_dual_gamma(r1, r2, r3, pr, taut)
        got, _ = e.debug_run_kernel("estimate_dual_gamma", [r1, r2, r3, *p], 6, [float(taut)])
        what = "%dx%d gamma %g %s" % (w, h, gamma, variant)
        if variant == "strict":
            for name, a, b in zip(("u1", "u2", "u3"), (g1, g2, g3), (r1, r2, r3)):
                _bits_equal(a, b, "%s %s" % (what, name))
            for k in range(6):
                _bits_equal(got[k], pr[k], "%s p%d" % (what, k))
            assert abs(err - err_ref) <= 1e-12 * abs(err_ref) + 1e-300, (what, err, err_ref)
        else:  # the default build's operation order (DESIGN §4.2): fp32 rounding apart
            for name, a, b in list(zip(("u1", "u2", "u3"), (g1, g2, g3), (r1, r2, r3))) + [("p%d" % k, got[k], pr[k]) for k in range(6)]:
                bad = np.abs(a.astype(np.float64) - b) > 2e-5 * (1 + np.abs(b.astype(np.float64)))
                assert not bad.any(), "%s %s: %d elements off, first at %s" % (what, name, bad.sum(), tuple(np.argwhere(bad)[0]))
            assert abs(err - err_ref) <= 1e-4 * abs(err_ref) + 1e-6, (what, err, err_ref)
    e.release()


# ---- strict build: the whole flow ----------------------------------------------------------------------------------------
def _fade(w, h):
    return cc.pair("fade_half", w, h)


# ((h, w), gamma, pair maker, knobs)
E2E = [((256, 256), 1.0, "bright", {}), ((256, 256), 0.1, "bright", {}), ((256, 340), 0.5, "fade", {}),
       ((97, 131), 1.0, "fade", {"lanes": 3}), ((97, 131), 2.0, "bright", {"median_filtering": 5, "median_interval": 7}),
       ((97, 131), 1.0, "plain", {"epsilon": 0.0, "iterations": 23}), ((1, 1), 1.0, "bright", {}), ((16, 16), 1.0, "bright", {}),
       ((17, 17), 0.3, "bright", {}), ((1080, 7), 1.0, "bright", {}), ((7, 1080), 1.0, "bright", {}),
       ((33, 33), 1.0, "bright", {"nscales": 2, "warps": 3})]


def _pair(kind, h, w, seed):
    if kind == "fade":
        return _fade(w, h)
    a, b, _ = synth.pair(h, w, seed)
    return (a, _brighter(b)) if kind == "bright" else (a, b)


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("case", range(len(E2E)))
def test_strict_flow_is_bit_exact(oracle, case, fused):
    (h, w), gamma, kind, params = E2E[case]
    a, b = _pair(kind, h, w, case)
    e = _new(w, h, gamma=gamma, **{**params, "fused": params.get("fused", fused)})
    flow = e.calc(a, b)
    iters, _ = e.tvl1_stats()
    pin.finish([pin.check(oracle, a, b, flow, iters, "%dx%d gamma %g %s %s" % (w, h, gamma, kind, params),
                          oracle_out=_reference(a, b, gamma, params))])
    e.release()


@pytest.mark.parametrize("lanes", [1, 3, 0])
def test_strict_clip_is_bit_exact(oracle, lanes):
    """pairs of a 340 x 256 clip whose brightness drifts, through one batch call, at 1 / 3 / automatic lanes and fused_k 3"""
    h, w = 256, 340
    fr = synth.stream(h, w, 5, seed=lanes)
    fr = np.stack([_brighter(f, 1.0 + 0.03 * i, 2.0 * i) for i, f in enumerate(fr)])
    e = _new(w, h, lanes=lanes, fused_k=3, gamma=0.8)
    flows = e.calc_batch(list(fr), step=1)
    pin.finish([pin.check(oracle, fr[j], fr[j + 1], flows[j], e.tvl1_pair_stats(j), "lanes %d pair %d" % (lanes, j),
                          oracle_out=T.tvl1_calc(fr[j], fr[j + 1], gamma=0.8)) for j in range(flows.shape[0])])
    e.release()


def test_strict_warm_start_is_bit_exact(oracle):
    h, w = 97, 131
    a, b, gt = synth.pair(h, w, 4)
    b = _brighter(b)
    start = (gt * 0.75).astype(np.float32)
    want = T.tvl1_calc(a, b, gamma=1.0, init=start)
    notes = []
    for fused in (1, 0):
        e = _new(w, h, gamma=1.0, use_initial_flow=1, fused=fused)
        flow = e.calc(a, b, flow=start.copy())
        iters, _ = e.tvl1_stats()
        notes.append(pin.check(oracle, a, b, flow, iters, "warm start, fused %d" % fused, oracle_out=want))
        e.release()
    pin.finish(notes)


# ---- both builds: the fused gamma kernel against the per-half-step schedule ---------------------------------------------------
def _drifting(h, w, n, seed):
    fr = synth.stream(h, w, n, seed=seed)
    return np.stack([_brighter(f, 1.0 + 0.01 * i, 0.5 * i) for i, f in enumerate(fr)])


def _schedules_agree(e, fr, what, flows=None):
    """e's batch through the fused gamma kernel at 1 / 3 / automatic lanes equals the per-half-step schedule pair by pair"""
    m = len(fr) - 1
    e.set("fused", 0)
    want = e.calc_batch(list(fr), step=1, flows=None if flows is None else flows.copy())
    logs = [e.tvl1_pair_stats(j) for j in range(m)]
    e.set("fused", 1)
    for lanes in (1, 3, 0):
        e.set("lanes", lanes)
        got = e.calc_batch(list(fr), step=1, flows=None if flows is None else flows.copy())
        _bits_equal(got, want, "%s, lanes %d" % (what, lanes))
        for j in range(m):
            assert np.array_equal(e.tvl1_pair_stats(j), logs[j]), (what, lanes, j)
    return want


@pytest.mark.parametrize("variant", VARIANTS)
def test_fused_equals_unfused_on_a_clip(variant):
    """a 64-frame 340 x 256 clip (63 pairs: more lanes than fit the parameter bank at automatic lanes) whose brightness drifts"""
    h, w = 256, 340
    fr = _drifting(h, w, 64, 100)
    e = _new(w, h, variant, gamma=0.8)
    _schedules_agree(e, fr, "340x256 clip")
    for knobs in (dict(fused_k=3, use_tma=0), dict(fused_k=1, use_tma=1)):  # tile-loop knobs: no effect on the gamma kernel
        for n, v in knobs.items():
            e.set(n, v)
        e.set("lanes", 0)
        _bits_equal(e.calc_batch(list(fr[:6]), step=1), e.set("fused", 0).calc_batch(list(fr[:6]), step=1), str(knobs))
        e.set("fused", 1)
    e.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_fused_equals_unfused_at_1080p(variant):
    h, w = 1080, 1920
    fr = _drifting(h, w, 4, 1)
    e = _new(w, h, variant, gamma=1.0)
    _schedules_agree(e, fr, "1080p batch")
    e.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_fused_equals_unfused_with_median_and_warm_starts(variant):
    h, w = 97, 131
    fr = _drifting(h, w, 6, 7)
    e = _new(w, h, variant, gamma=2.0, median_filtering=5, median_interval=7)
    _schedules_agree(e, fr, "median")
    e.set("median_filtering", 0).set("use_initial_flow", 1)
    starts = (np.random.default_rng(3).standard_normal((5, h, w, 2)) * 2).astype(np.float32)
    _schedules_agree(e, fr, "warm starts", flows=starts)
    e.release()


# ---- default build ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma", [0.1, 1.0])
def test_default_is_near_the_restatement(gamma):
    h, w = 256, 340
    a, b, _ = synth.pair(h, w, 3)
    b = _brighter(b)
    e = _new(w, h, "default", gamma=gamma)
    ref = e.calc(a, b)
    _bits_equal(e.set("fused", 0).calc(a, b), ref, "gamma %g, unfused" % gamma)
    o = T.tvl1_calc(a, b, gamma=gamma)[0]
    epe = np.hypot(*(ref.astype(np.float64) - o).transpose(2, 0, 1))
    print("default build with gamma %g vs the restatement: AEE %.3g, p99.9 EPE %.3g px" % (gamma, epe.mean(), np.percentile(epe, 99.9)))
    assert epe.mean() <= AEE_TOL, epe.mean()
    e.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_batches_equal_single_pairs(variant):
    import torch
    h, w = 97, 131
    fr = synth.stream(h, w, 8, seed=11)
    fr = np.stack([_brighter(f, 1.0 + 0.02 * i, 3.0 * i) for i, f in enumerate(fr)])
    e = _new(w, h, variant, gamma=1.0)
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


def test_every_entry_point_takes_gamma():
    """the float, planar, quantised, PNG and colour-chain calls of one gamma handle agree with its calc_batch"""
    import torch
    import denseflow_b200 as d
    from test_jpeg_encode_gpu import _colour, imencode
    h, w, bound = 96, 128, 20
    gray = synth.stream(h, w, 6, seed=5)
    gray = np.stack([_brighter(f, 1.0 + 0.04 * i, 4.0 * i) for i, f in enumerate(gray)])
    bgr = _colour(gray)
    e = d.create("tvl1", 0, w, h)
    e.set("gamma", 1.0)
    flows = e.calc_batch(list(gray), step=1)
    plain = d.create("tvl1", 0, w, h)
    assert (plain.calc_batch(list(gray), step=1) != flows).any(), "gamma did not change the flow"
    plain.release()
    _bits_equal(e.calc_batch_planes(list(gray), step=1), flows.transpose(0, 3, 1, 2), "calc_batch_planes")
    dev = torch.from_numpy(np.ascontiguousarray(gray)).cuda()
    _bits_equal(e.calc_batch_device_planes(dev, step=1).cpu().numpy(), flows.transpose(0, 3, 1, 2), "calc_batch_device_planes")
    qx, qy = e.calc_batch(list(gray), step=1, bound=bound)
    for j in range(flows.shape[0]):
        rx, ry = R_quantise(flows[j], bound)
        assert np.array_equal(qx[j], rx) and np.array_equal(qy[j], ry), j
    # the colour chains convert to gray first: compare with calc_batch of their own gray frames
    g2 = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]
    f2 = e.calc_batch(g2, step=1)
    _bits_equal(e.process_bgr_batch_planes(bgr, step=1), f2.transpose(0, 3, 1, 2), "process_bgr_batch_planes")
    q2x, q2y = e.calc_batch(g2, step=1, bound=bound)
    e.set("jpeg_exact", 1)
    for i, (jx, jy) in enumerate(e.process_bgr_batch(bgr, step=1, bound=bound)):
        assert jx == imencode(q2x[i]) and jy == imencode(q2y[i]), i
    for i, png in enumerate(e.calc_batch_png(list(gray), step=1)):  # the flow map image of calc_batch's flow, losslessly
        img = cv2.imdecode(np.frombuffer(bytes(png), np.uint8), cv2.IMREAD_COLOR)
        assert np.array_equal(img, cv_restate.flow_to_png_image(flows[i])[0]), i
    e.release()


def R_quantise(flow, bound):
    from oracle import pyoracle
    return pyoracle.quantise(flow, bound)


# ---- parameter state ---------------------------------------------------------------------------------------------------------
NOT_FINITE = [float("nan"), float("inf"), float("-inf")]


@pytest.mark.parametrize("variant", VARIANTS)
def test_parameter_table(variant):
    import denseflow_b200 as d
    e = d.OpticalFlowDual_TVL1.create(0, 64, 64, variant)
    L = _lib.load(variant)
    assert e.get("gamma") == 0
    for v in (0.5, 0.0, 1e-7, 3.0, 1e6):
        e.set("gamma", v)
        assert e.get("gamma") == v
    e.set("gamma", 0.25)
    for v in NOT_FINITE + [-1e-9, -0.5, -1e10]:
        assert L.dfb_set_param(e._h, b"gamma", float(v)) == _lib.DFB_ERR_INVALID_ARG, v
        assert L.dfb_last_error(e._h).decode() == "bad parameter gamma", v
        assert e.get("gamma") == 0.25, v
    e.release()
    f = d.FarnebackOpticalFlow.create(0, 64, 64, variant)
    assert L.dfb_set_param(f._h, b"gamma", 0.5) == _lib.DFB_ERR_INVALID_ARG
    assert L.dfb_last_error(f._h).decode() == "bad parameter gamma"
    f.release()


@pytest.mark.parametrize("variant", VARIANTS)
def test_gamma_off_again_equals_a_fresh_handle(variant):
    h, w = 97, 131
    fr = synth.stream(h, w, 4, seed=3)
    fresh = _new(w, h, variant)
    want = fresh.calc_batch(list(fr), step=1)
    want_iters = [fresh.tvl1_pair_stats(j) for j in range(3)]
    fresh.release()
    e = _new(w, h, variant, gamma=2.0)
    on = e.calc_batch(list(fr), step=1)
    assert (on != want).any(), "gamma did not change the flow"
    e.set("gamma", 0)
    _bits_equal(e.calc_batch(list(fr), step=1), want, "gamma set back to 0")
    assert all(np.array_equal(e.tvl1_pair_stats(j), want_iters[j]) for j in range(3))
    e.release()


def test_gamma_handle_beside_default_handle():
    h, w = 256, 340
    fr = synth.stream(h, w, 6, seed=6)
    plain = _new(w, h, "default")
    want = plain.calc_batch(list(fr), step=1)
    gam = _new(w, h, "default", gamma=1.0)
    gam_alone = gam.calc_batch(list(fr), step=1)
    got, errors = {}, []

    def run_gamma():
        try:
            for i in range(2):
                got["gamma%d" % i] = gam.calc_batch(list(fr), step=1)
        except Exception as ex:  # surfaced below
            errors.append(ex)

    t = threading.Thread(target=run_gamma)
    t.start()
    plain_runs = [plain.calc_batch(list(fr), step=1) for _ in range(2)]
    t.join()
    assert not errors, errors
    for i, f in enumerate(plain_runs):
        _bits_equal(f, want, "default handle, run %d beside the gamma handle" % i)
    for i in range(2):
        _bits_equal(got["gamma%d" % i], gam_alone, "gamma handle, run %d beside the default handle" % i)
    plain.release()
    gam.release()
