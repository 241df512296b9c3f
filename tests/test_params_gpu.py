"""Both engines away from the create() defaults, and the parameter values set() refuses.

* TV-L1 end to end on 3-frame streams at 340 x 256 (levels small enough to stay resident on chip) and 131 x 97, one case per
  parameter plus combinations.  Strict build: flows and per-(scale, warp) logs equal the oracle's at the full parameter set,
  fused (1 lane and the automatic count) and unfused.  Default build: finite flows, fused equal to unfused bit for bit, and
  the 0.01 px / 5 % iteration contract where the pair converges (0.05 px at lambda = 1, see AEE_TOL_LAMBDA_1; a pair at
  the cap everywhere must have the oracle's schedule; its flow is chaotic under rounding and the strict pin is its
  guarantee).
* The stand-alone primal / dual kernels and the fused kernel's chunk and upsample stages at other l_t, taut, theta and
  scale steps (tests/test_params_cpu.py checks the float64 bounds there first).
* Deep pyramids: 16 levels at 1920 x 1080 and 3840 x 2160 (the capacity the frame slots and lanes are allocated for), and
  16 scales x 16 warps at 340 x 256 (13 x 16 log entries).
* One 3840 x 2160 handle taken through a sequence of settings, every entry point equal to a fresh handle's bytes; the
  iteration log a call leaves behind describes that call after a later set().
* Farneback at other poly_sigma and num_iters.
* set() refuses NaN, the infinities, fractions of counts and values out of range for every parameter, and keeps the old value.
* The fused kernel's phase profiler keeps its per-scale slots apart when nscales > 8."""
import ctypes as C
import math

import numpy as np
import pytest

import test_tvl1_fused_stages_gpu as fs
import tvl1_pin as pin
import tvl1_ref64 as r64
from denseflow_b200 import _lib, synth
from tvl1_cases import chunk_inputs

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
AEE_TOL = 0.01  # px, BASELINE.json north_star
# lambda = 1 (l_t = 0.3, twice the default's 0.045 at theta 0.3 and 0.15 at theta 1): the stiffer data term amplifies the
# default build's rounding.  Measured on an H100 80GB HBM3 at a 700 W power limit: AEE 2.5e-3 px on the pair whose schedule equals the oracle's,
# and 1.0e-2 to 2.8e-2 px on the pairs where a convergence check went the other way (iteration totals within 3 %).  The
# strict pin is the guarantee there; this bound guards against worse.
AEE_TOL_LAMBDA_1 = 0.05
ORACLE_KEYS = ("tau", "lambda", "theta", "nscales", "warps", "epsilon", "iterations", "scale_step")
TVL1_DEFAULTS = dict(tau=0.25, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300, scale_step=0.8, fused=1, fused_k=8,
                     lanes=0, **{"lambda": 0.15})
_handles = {}
_oracle = {}


@pytest.fixture(scope="module", autouse=True)
def _release_handles():
    """the handles' device memory goes back before the next test module runs"""
    yield
    for e in _handles.values():
        e.release()
    _handles.clear()
    _oracle.clear()
    import torch
    torch.cuda.empty_cache()


def _handle(alg, variant, w, h):
    key = (alg, variant, w, h)
    if key not in _handles:
        import denseflow_b200 as d
        _handles[key] = d.create(alg, 0, w, h, variant)
    return _handles[key]


def _configure(e, params, defaults=TVL1_DEFAULTS):
    for k, v in dict(defaults, **params).items():
        e.set(k, v)
    return e


def _oracle_params(oracle, params):
    return oracle.tvl1_params(**{k: v for k, v in params.items() if k in ORACLE_KEYS})


def _oracle_out(oracle, a, b, params):
    key = (a.shape, synth.sha1(a), synth.sha1(b), tuple(sorted((k, v) for k, v in params.items() if k in ORACLE_KEYS)))
    if key not in _oracle:
        big = a.size > 1 << 20
        if big:
            oracle.lib().orc_set_num_threads(oracle.usable_cores())
        try:
            _oracle[key] = oracle.tvl1_calc(a, b, _oracle_params(oracle, params), return_iters=True, return_errors=True)
        finally:
            if big:
                oracle.lib().orc_set_num_threads(min(8, oracle.usable_cores()))
    return _oracle[key]


def _same(got, want, name):
    diff = np.any(got != want, axis=-1) if got.ndim == 3 else got != want
    assert not diff.any(), "%s: %d pixels differ, first at %s" % (name, diff.sum(), tuple(np.argwhere(diff)[0]))


# ---- end-to-end grid ----------------------------------------------------------------------------------------------------
GRID = [{"tau": 0.1}, {"tau": 0.5}, {"lambda": 0.0}, {"lambda": 0.05}, {"lambda": 1.0}, {"theta": 0.05}, {"theta": 1.0},
        {"scale_step": 0.3}, {"scale_step": 0.5}, {"scale_step": 0.7}, {"nscales": 9}, {"warps": 9}, {"epsilon": 1.0},
        {"epsilon": 0.0, "iterations": 30}, {"iterations": 1}, {"iterations": 3}, {"fused_k": 3},
        {"theta": 1.0, "scale_step": 0.5}, {"lambda": 1.0, "fused_k": 3}, {"tau": 0.5, "theta": 0.05, "lambda": 1.0, "warps": 2},
        {"scale_step": 0.3, "nscales": 16, "warps": 2, "fused_k": 5}]
SHAPES = [(340, 256), (131, 97)]


def _grid_id(p):
    return "-".join("%s%g" % kv for kv in p.items())


@pytest.mark.parametrize("variant", VARIANTS)  # varies fastest: both builds share one oracle run per case
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%d" % s for s in SHAPES])
@pytest.mark.parametrize("params", GRID, ids=[_grid_id(p) for p in GRID])
def test_tvl1_off_defaults(oracle, params, shape, variant):
    w, h = shape
    fr = synth.stream(h, w, 3, seed=w + len(params))
    pairs = [(fr[0], fr[1]), (fr[1], fr[2])]
    e = _handle("tvl1", variant, w, h)
    tag = "%s %dx%d %s" % (variant, w, h, params)
    runs = {}
    for fused, lanes in ((1, 1), (1, 0), (0, 0)):
        _configure(e, dict(params, fused=fused, lanes=lanes))
        flows = e.calc_batch(list(fr), step=1)
        runs[(fused, lanes)] = (flows, [e.tvl1_pair_stats(j) for j in range(2)])
    _configure(e, {})
    notes = []
    for j, (a, b) in enumerate(pairs):
        ref, log, errs = _oracle_out(oracle, a, b, params)
        if variant == "strict":
            for (fused, lanes), (flows, iters) in runs.items():
                notes.append(pin.check(oracle, a, b, flows[j], iters[j], "%s pair %d fused %d lanes %d" % (tag, j, fused, lanes),
                                       oracle_out=(ref, log, errs)))
            continue
        for key in ((1, 0), (0, 0)):
            _same(runs[key][0][j], runs[(1, 1)][0][j], "%s pair %d fused/lanes %s vs fused lanes 1" % (tag, j, key))
            assert np.array_equal(runs[key][1][j], runs[(1, 1)][1][j]), (tag, j, key)
        flow, iters = runs[(1, 1)][0][j], runs[(1, 1)][1][j]
        assert np.isfinite(flow).all(), tag
        cap = params.get("iterations", 300)
        levels = len(oracle.tvl1_level_sizes(w, h, _oracle_params(oracle, params)))
        if (log[:levels] == cap).all():
            assert np.array_equal(iters, log[:levels]), (tag, j, iters.tolist(), log.tolist())
        else:
            aee = synth.aee(flow, ref)
            print("%s pair %d: AEE %.3e px, iterations %d (oracle %d)" % (tag, j, aee, iters.sum(), log.sum()))
            assert aee <= (AEE_TOL_LAMBDA_1 if params.get("lambda", 0) >= 1 else AEE_TOL), (tag, j, aee)
            assert abs(int(iters.sum()) - int(log.sum())) <= 0.05 * log.sum(), (tag, j, iters.sum(), log.sum())
    pin.finish(notes)


# ---- stages at other constants ------------------------------------------------------------------------------------------
STAGE_CONSTS = [(0.25, 0.0, 0.3), (0.25, 0.15, 0.05), (0.25, 1.0, 0.3), (0.25, 1.0, 1.0), (1.25, 0.15, 0.05), (0.1, 0.05, 1.0)]


@pytest.mark.parametrize("variant", VARIANTS)
def test_primal_and_dual_kernels_off_defaults(oracle, variant):
    """estimate_u and estimate_dual at the l_t, taut and theta of (tau, lambda, theta) above: strict equal to the oracle's
    building blocks, default within the float64 bounds"""
    L = oracle.lib()
    e = _handle("tvl1", variant, 64, 64)
    for j, (w, h) in enumerate([(37, 53), (131, 97), (270, 61)]):
        ix, iy, g, rc, u1, u2, *p = chunk_inputs(w, h, 40 + j)
        for tau, lam, theta in STAGE_CONSTS:
            l_t, taut, th = fs.consts(tau, lam, theta)
            tag = "%dx%d l_t %g taut %g theta %g" % (w, h, l_t, taut, th)
            r1, r2 = u1.copy(), u2.copy()
            err_ref = L.orc_tvl1_estimate_u(ix, iy, g, rc, *p, r1, r2, w, h, l_t, th, 1)
            (g1, g2), err = e.debug_run_kernel("estimate_u", [ix, iy, g, rc, *p, u1, u2], 2, [float(l_t), float(th), 1])
            pr = [q.copy() for q in p]
            L.orc_tvl1_estimate_dual(r1, r2, *pr, w, h, taut)
            got, _ = e.debug_run_kernel("estimate_dual", [r1, r2, *p], 4, [float(taut)])
            if variant == "strict":
                fs._check(tag + " u1", g1, r1)
                fs._check(tag + " u2", g2, r2)
                assert abs(err - err_ref) <= 1e-12 * abs(err_ref), (tag, err, err_ref)
                for k in range(4):
                    fs._check("%s p%d" % (tag, k), got[k], pr[k])
                continue
            ref = r64.primal(ix, iy, g, rc, u1, u2, *p, l_t, th)
            for name, bad in zip(("u1", "u2"), r64.within_primal(g1, g2, ref)):
                assert not bad.any(), "%s %s: %d elements outside the float64 bound, first at %s" % (tag, name, bad.sum(), tuple(np.argwhere(bad)[0]))
            s, b = r64.convergence_sum(u1, u2, g1, g2, ref)
            assert abs(err - s) <= b, (tag, err, s, b)
            for k, (v, b) in enumerate(r64.dual(r1, r2, *p, taut)):
                bad = ~(np.abs(got[k].astype(np.float64) - v) <= b)
                assert not bad.any(), "%s p%d: %d elements outside the float64 bound, first at %s" % (tag, k, bad.sum(), tuple(np.argwhere(bad)[0]))


@pytest.mark.parametrize("variant", VARIANTS)
def test_chunks_off_defaults(oracle, variant):
    """the fused chunk loop with the handle's tau, lambda and theta set: strict equal to oracle_chunks at those constants,
    default equal to the stand-alone kernels"""
    shapes = [(340, 256), (131, 97), (250, 61), (16, 16)]
    for j, (tau, lam, theta) in enumerate(STAGE_CONSTS):
        for i, (w, h) in enumerate(shapes):
            kk = fs.KS[(i + j) % len(fs.KS)]
            fs.run_chunks(oracle, variant, w, h, kk, 2, fs.CONFIGS[(5 * j + 3 * i) % len(fs.CONFIGS)], 900 + 10 * j + i, tau, lam, theta)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("step", [0.5, 0.7])
def test_upsample_off_defaults(oracle, variant, step):
    """the fused upsample stage multiplies by the handle's float(1 / scale_step), between every two levels of that pyramid"""
    e = fs._engine(variant)
    mul = 1.0 / step
    keep = e.get("scale_step")
    try:
        e.set("scale_step", step)
        for w, h in ((1920, 1080), (340, 256), (131, 97)):
            lv = oracle.tvl1_level_sizes(w, h, oracle.tvl1_params(nscales=16, scale_step=step))
            for s, ((dw, dh), (sw, sh)) in enumerate(zip(lv, lv[1:])):
                lanes = 1 + 2 * (s % 2)
                ins = [[(np.random.default_rng(sw * 10 + i + c).standard_normal((sh, sw)) * 4).astype(np.float32) for c in range(2)]
                       for i in range(lanes)]
                got, _ = e.debug_run_kernel("tvl1_upsample", [fs._stack([c[k] for c in ins]) for k in range(2)], 2, [dw, dh, lanes],
                                            out_shape=(dh * lanes, dw))
                for i in range(lanes):
                    for c in range(2):
                        want, fx, fy = fs._ref_upsample(ins[i][c], dw, dh, mul)
                        g = fs._split(got[c], lanes)[i]
                        tag = "step %g %dx%d -> %dx%d lane %d u%d" % (step, sw, sh, dw, dh, i, c + 1)
                        if variant == "strict":
                            fs._check(tag, g, want)
                        else:
                            v, b = r64.upsample(ins[i][c], dw, dh, fx, fy, mul)
                            bad = ~(np.abs(g.astype(np.float64) - v) <= b)
                            assert not bad.any(), (tag, bad.sum(), tuple(np.argwhere(bad)[0]))
    finally:
        e.set("scale_step", keep)


# ---- deep pyramids ------------------------------------------------------------------------------------------------------
DEEP = [((1920, 1080), dict(nscales=16, warps=1, iterations=10, epsilon=0.0)),
        ((3840, 2160), dict(nscales=16, warps=1, iterations=10, epsilon=0.0)),
        ((340, 256), dict(nscales=16, warps=16, iterations=20))]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", range(len(DEEP)), ids=["%dx%d" % c[0] for c in DEEP])
def test_deep_pyramids(oracle, case, variant):
    (w, h), params = DEEP[case]
    a, b, _ = synth.pair(h, w, case)
    ref, log, errs = _oracle_out(oracle, a, b, params)
    sizes = oracle.tvl1_level_sizes(w, h, _oracle_params(oracle, params))
    e = _handle("tvl1", variant, w, h)
    tag = "%s %dx%d %s" % (variant, w, h, params)
    flows, notes = [], []
    for fused in (1, 0):
        _configure(e, dict(params, fused=fused))
        flow = e.calc(a, b)
        iters, got_sizes = e.tvl1_stats()
        assert got_sizes == sizes, (tag, got_sizes)
        assert iters.shape == (len(sizes), params["warps"]) and np.array_equal(e.tvl1_pair_stats(0), iters), tag
        if variant == "strict":
            notes.append(pin.check(oracle, a, b, flow, iters, "%s fused %d" % (tag, fused), oracle_out=(ref, log, errs)))
        else:
            assert np.isfinite(flow).all(), tag
            if "epsilon" in params:
                assert (iters == params["iterations"]).all(), (tag, iters.tolist())
        flows.append(flow)
    _configure(e, {})
    if variant == "default":
        _same(flows[0], flows[1], tag + " fused vs unfused")
    pin.finish(notes)


# ---- one handle, parameters changed between calls -----------------------------------------------------------------------
SEQUENCE = [{}, {"scale_step": 0.5, "nscales": 16}, {}, {"warps": 16, "iterations": 40}, {"fused_k": 3}, {"lambda": 1.0, "theta": 1.0},
            {"scale_step": 0.3, "fused": 0}, {"lanes": 1, "nscales": 3, "tau": 0.5}, {}]


@pytest.mark.parametrize("variant", VARIANTS)
def test_one_handle_through_a_parameter_sequence(variant):
    """Every call on a 3840 x 2160 handle whose parameters keep changing gives the bytes of a fresh handle created with the
    current parameters: geometry, tensor maps and constants are never kept across a set().  The batches have 5 pairs on 3
    lanes.  The iteration logs of a call still describe it after the next step's set() calls."""
    import torch
    import denseflow_b200 as d
    h, w = 360, 640
    fr = synth.stream(h, w, 6, seed=21)
    big_a, big_b, _ = synth.pair(2160, 3840, 5)
    e = _handle("tvl1", variant, 3840, 2160)
    base = dict(TVL1_DEFAULTS, lanes=3)
    prev = None
    for i, step in enumerate(SEQUENCE):
        _configure(e, step, base)
        if prev is not None:  # the previous step's logs, read after this step's set() calls
            assert [e.tvl1_pair_stats(j).tolist() for j in range(5)] == prev, (variant, i)
        tag = "%s step %d %s" % (variant, i, step)
        fresh = _configure(d.OpticalFlowDual_TVL1.create(0, w, h, variant), step, base)
        try:
            _same(e.calc(fr[0], fr[1]), fresh.calc(fr[0], fr[1]), tag + " calc")
            assert np.array_equal(e.tvl1_stats()[0], fresh.tvl1_stats()[0]), tag
            want = fresh.calc_batch(list(fr), step=1)
            want_logs = [fresh.tvl1_pair_stats(j).tolist() for j in range(5)]
            got = e.calc_batch(list(fr), step=1)
            _same(got, want, tag + " calc_batch")
            assert [e.tvl1_pair_stats(j).tolist() for j in range(5)] == want_logs, tag
            dev = e.calc_batch_device(torch.from_numpy(np.stack(fr)).cuda(), step=1)
            torch.cuda.synchronize()
            _same(dev.cpu().numpy(), want, tag + " calc_batch_device")
            prev = [e.tvl1_pair_stats(j).tolist() for j in range(5)]
            assert prev == want_logs, tag
        finally:
            fresh.release()
        if i in (0, 1):  # frames of the handle's full size: every level of the allocated pyramid in use at 0.8
            big = e.calc(big_a, big_b)
            fresh = _configure(d.OpticalFlowDual_TVL1.create(0, 3840, 2160, variant), step, base)
            try:
                _same(big, fresh.calc(big_a, big_b), tag + " 3840x2160 calc")
            finally:
                fresh.release()
            prev = None
    _configure(e, {})


@pytest.mark.parametrize("fused", [1, 0])
def test_stats_describe_the_call_that_ran(oracle, fused):
    """tvl1_stats / tvl1_pair_stats lay the log out with the warps of the call that wrote it, not of a later set()"""
    h, w = 97, 131
    fr = synth.stream(h, w, 3, seed=4)
    e = _handle("tvl1", "strict", w, h)
    params = dict(warps=3, nscales=4, iterations=50)
    _configure(e, dict(params, fused=fused))
    e.calc(fr[0], fr[1])
    e.set("warps", 5).set("nscales", 2)
    iters, sizes = e.tvl1_stats()
    _, log, _ = _oracle_out(oracle, fr[0], fr[1], params)
    assert iters.shape == (4, 3) and np.array_equal(iters, log), (iters.tolist(), log.tolist())
    assert sizes == oracle.tvl1_level_sizes(w, h, _oracle_params(oracle, params))
    _configure(e, dict(params, fused=fused))
    e.calc_batch(list(fr), step=1)
    e.set("warps", 7)
    for j in range(2):
        _, log, _ = _oracle_out(oracle, fr[j], fr[j + 1], params)
        assert np.array_equal(e.tvl1_pair_stats(j), log), (j, e.tvl1_pair_stats(j).tolist(), log.tolist())
    _configure(e, {})


# ---- Farneback ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("shape", [(340, 256), (131, 97)], ids=["340x256", "131x97"])
def test_farneback_off_defaults(oracle, shape, variant):
    w, h = shape
    a, b, _ = synth.pair(h, w, 3)
    e = _handle("farn", variant, w, h)
    try:
        for sigma in (0.8, 1.5, 2.0):
            for iters in (1, 25):
                tag = "farn %s %dx%d poly_sigma %g num_iters %d" % (variant, w, h, sigma, iters)
                e.set("poly_sigma", sigma).set("num_iters", iters)
                flow = e.calc(a, b)
                if variant == "strict":
                    _same(flow, oracle.farn_calc(a, b, oracle.farn_params(poly_sigma=sigma, num_iters=iters)), tag + " vs orc_farn_calc")
                else:
                    assert np.isfinite(flow).all(), tag
    finally:
        e.set("poly_sigma", 1.1).set("num_iters", 10)


# ---- refusals -----------------------------------------------------------------------------------------------------------
NAN, INF = math.nan, math.inf
NOT_FINITE = [NAN, INF, -INF]
FLAG = NOT_FINITE + [0.5, 2, -1]
REFUSED = {
    "tvl1": {"tau": NOT_FINITE + [0, -0.0, -0.25, -1e-300], "lambda": NOT_FINITE + [-0.15, -1e-300],
             "theta": NOT_FINITE + [0, -0.3], "nscales": NOT_FINITE + [0, -1, 17, 2.5, 1e10], "warps": NOT_FINITE + [0, 17, 2.5],
             "epsilon": NOT_FINITE, "iterations": NOT_FINITE + [0, -3, 2.5, 1e10, 2.0 ** 31],
             "scale_step": NOT_FINITE + [0, -0.5, 0.81, 1.0], "fused": FLAG, "fused_k": NOT_FINITE + [0, 9, 2.5, -1],
             "time_kernels": FLAG, "use_tma": FLAG, "lanes": NOT_FINITE + [-1, 65, 2.5]},
    "farn": {"num_levels": NOT_FINITE + [-1, 6, 2.5], "num_iters": NOT_FINITE + [0, -1, 2.5, 1e10],
             "poly_sigma": NOT_FINITE + [0, -1.1], "pyr_scale": NOT_FINITE + [0, 0.25], "win_size": NOT_FINITE + [15, 13.5],
             "poly_n": NOT_FINITE + [7], "time_kernels": FLAG},
}
ACCEPTED = {
    "tvl1": [("nscales", 1), ("nscales", 16), ("warps", 1), ("warps", 16), ("fused_k", 1), ("fused_k", 8), ("lanes", 64), ("lanes", 0),
             ("lambda", 0), ("epsilon", 0), ("epsilon", -1), ("iterations", 1), ("iterations", 2 ** 31 - 1), ("scale_step", 0.8),
             ("scale_step", 0.05), ("tau", 1e-3), ("theta", 5.0), ("fused", 0)],
    "farn": [("num_levels", 0), ("num_levels", 5), ("num_iters", 1), ("poly_sigma", 0.8), ("pyr_scale", 0.5), ("win_size", 13),
             ("poly_n", 5)],
}


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_set_refuses_bad_values_and_keeps_the_old_one(alg, variant):
    """set/get only: nothing is launched with a refused value"""
    e = _handle(alg, variant, 64, 64)
    L = _lib.load(variant)
    for name, v in ACCEPTED[alg]:
        assert L.dfb_set_param(e._h, name.encode(), float(v)) == _lib.DFB_OK, (name, v)
        if name != "pyr_scale":
            assert e.get(name) == v, (name, v, e.get(name))
    for name, values in REFUSED[alg].items():
        for v in values:
            before = e.get(name)
            assert L.dfb_set_param(e._h, name.encode(), float(v)) == _lib.DFB_ERR_INVALID_ARG, (alg, name, v)
            assert L.dfb_last_error(e._h).decode() == "bad parameter " + name, (alg, name, v)
            after = C.c_double()
            assert L.dfb_get_param(e._h, name.encode(), C.byref(after)) == _lib.DFB_OK
            assert after.value == before, (alg, name, v, after.value, before)
    # names of removed engine knobs: a handle refuses them like any name it does not know
    removed = ("use_tma",) if alg == "farn" else ("flag_sync", "prefetch", "serial_launches")
    before = {n: e.get(n) for n in REFUSED[alg]}
    for name in removed:
        for v in (0, 1):
            assert L.dfb_set_param(e._h, name.encode(), float(v)) == _lib.DFB_ERR_INVALID_ARG, (alg, name, v)
            assert L.dfb_last_error(e._h).decode() == "bad parameter " + name, (alg, name, v)
        assert L.dfb_get_param(e._h, name.encode(), C.byref(C.c_double())) == _lib.DFB_ERR_INVALID_ARG, (alg, name)
    assert {n: e.get(n) for n in REFUSED[alg]} == before
    e.release()
    del _handles[(alg, variant, 64, 64)]


# ---- phase profiler -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
def test_profiler_per_scale_slots_with_more_than_eight_scales(variant):
    """epsilon 0, 23 iterations in chunks of at most 8: every warp of every scale runs 3 chunks (8 + 8 + 7); 12 levels
    of 340 x 256, so scales 8..11 exist and must not land in the chunk counts of scales 0..3"""
    h, w = 256, 340
    a, b, _ = synth.pair(h, w, 2)
    e = _handle("tvl1", variant, w, h)
    params = dict(epsilon=0.0, iterations=23, fused_k=8, lanes=1, nscales=12)
    _configure(e, params)
    e.calc(a, b)
    iters, sizes = e.tvl1_stats()
    assert len(sizes) == 12 and (iters == 23).all()
    ph = e.phase_ns()
    _configure(e, {})
    assert ph["chunks_per_scale"] == [3 * params.get("warps", 5)] * 8, ph["chunks_per_scale"]
    assert all(t > 0 for t in ph["tiles_per_scale"]) and sum(ph["tiles_per_scale"]) <= ph["tiles"], ph
