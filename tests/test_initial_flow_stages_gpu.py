"""The start of a warm solve (`use_initial_flow`, DESIGN §1) as a stage of its own, through the `tvl1_initial_flow` and
`farn_initial_flow` stages of dfb_debug_run_kernel (the engines' own load_initial_flow / launch_flow_init):

* TV-L1: every level of every lane's start pyramid.  Strict build: equal to tests/tvl1_restate.tvl1_init_pyramid bit
  for bit.  Default build: level 0 is the start itself, every coarser level within the float64 bound of
  tvl1_ref64.upsample(level above, ..., float(scale_step)), element by element.
* Farneback: the coarsest level's start.  Strict build: equal to farn_restate.farn_start (orc_resize_linear x
  float(pyrScale^k), as in farn_restate.farn_calc) bit for bit.  Default build: within farn_ref64.level_start's bound.

Covered: the frame shapes of tests/farn_cases.py and 4K, geometry_cases' tiny frames, small planes, strips and the sizes at
and just below every level cut; TV-L1 at the nscales / scale_step pairs of the CPU pyramid tests, Farneback at num_levels
0 / 1 / 3 / 5; the start as a float2 field (step 2) or two planes (step 1), dense or with a padded row pitch; TV-L1 on 1,
3, 16, 17 and 40 lanes (the copy kernel takes 16 starts per launch) and Farneback on 1, 3 and 8 pairs; smooth, i.i.d.,
signed-zero and far-outside starts (up to 4x the frame size), a different one per lane.  The lane pyramids and the start
buffers' padding hold NaN before the stage runs."""
import numpy as np
import pytest

import farn_cases as fc
import farn_ref64 as f64
import farn_restate as R
import geometry_cases as gc
import tvl1_ref64 as t64
import tvl1_restate as T
from test_initial_flow_cpu import PYRAMIDS, smooth_field

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
F = np.float32
KINDS = ["smooth", "iid", "zeros", "far"]
BIG = (3840, 2160)
SMALL = (400, 400)  # the handle of every shape that fits it; lanes sized for it, so 40 of them stay small
FRAMES = fc.FRAME_SHAPES + [BIG]
TVL1_PARAMS = sorted({(n, s) for _, _, n, s in PYRAMIDS})  # 1, 5 and 16 levels; 0.8, 0.5 and 0.3
FARN_LEVELS = [0, 1, 3, 5]
# the sizes at and below every level cut of both engines (the Farneback cuts go up to 1024 x 1024)
CUTS = sorted(set(gc.TVL1_CUTS + gc.FARN_CUTS))
GROUPS = {"tiny": gc.TINY, "small": gc.STAGE_SMALL, "strips": gc.STAGE_STRIPS, "cuts": CUTS}


def start(kind, w, h, seed):
    """one lane's start [h, w, 2]"""
    rng = np.random.default_rng(seed)
    if kind == "smooth":
        return smooth_field(h, w, seed, amp=6.0)
    if kind == "iid":
        return rng.normal(0.0, 3.0, (h, w, 2)).astype(F)
    if kind == "zeros":  # +0 and -0, and a few values so that every lane differs
        f = np.where(rng.random((h, w, 2)) < 0.5, F(-0.0), F(0.0)).astype(F)
        some = rng.random((h, w, 2)) < 0.05
        f[some] = rng.normal(0.0, 1.0, some.sum())
        return f
    if kind == "far":  # far outside the frame: up to 4x its size
        return (rng.uniform(-4.0, 4.0, (h, w, 2)) * np.array([w, h])).astype(F)
    raise ValueError(kind)


def layouts(w):
    """(step, pitch in floats): two planes or a float2 field, each dense (0) and with rows padded by an odd count"""
    return [(1, 0), (1, w + 37), (2, 0), (2, 2 * w + 37)]


def _bits_equal(got, want, what):
    got, want = np.ascontiguousarray(got, F), np.ascontiguousarray(want, F)
    bad = got.view(np.int32) != want.view(np.int32)
    assert not bad.any(), "%s: %d of %d differ, first at %s: %r vs %r" % (what, bad.sum(), bad.size, tuple(np.argwhere(bad)[0]),
                                                                      got[bad][0], want[bad][0])


def _within(got, ref, what):
    v, b = ref
    bad = ~(np.abs(got.astype(np.float64) - v) <= b)
    assert not bad.any(), "%s: %d elements outside the float64 bound, first at %s: got %r, float64 %r, bound %r" % (
        what, bad.sum(), tuple(np.argwhere(bad)[0]), got[bad][0], v[bad][0], b[bad][0])


_handles = {}


def _handle(alg, variant, size):
    import denseflow_b200 as d
    key = (alg, variant, size)
    if key not in _handles:
        _handles[key] = d.create(alg, 0, size[0], size[1], variant)
    return _handles[key]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for e in _handles.values():
        e.release()
    _handles.clear()


def _size_for(w, h):
    return SMALL if w <= SMALL[0] and h <= SMALL[1] else BIG


# ---- TV-L1 ---------------------------------------------------------------------------------------------------------------------
def tvl1_case(oracle, e, variant, w, h, nscales, scale_step, starts, step, pitch, what):
    e.set("nscales", nscales).set("scale_step", scale_step)
    lv = oracle.tvl1_level_sizes(w, h, oracle.tvl1_params(nscales=nscales, scale_step=scale_step))
    n = len(starts)
    x = np.concatenate([s[..., 0] for s in starts])
    y = np.concatenate([s[..., 1] for s in starts])
    sizes = [n * lw * lh for lw, lh in lv]
    outs, _ = e.debug_run_kernel("tvl1_initial_flow", [x, y], 2, [step, pitch, n], out_shape=(sum(sizes),))
    # each output holds level after level, a level the lanes' planes one after the other
    levels = [[o[a:a + m].reshape(n, lh, lw) for a, m, (lw, lh) in zip(np.cumsum([0] + sizes), sizes, lv)] for o in outs]
    finv = F(1.0 / scale_step)
    for i, init in enumerate(starts):
        got = [[lev[i] for lev in levels[c]] for c in (0, 1)]
        tag = "%s %dx%d nscales %d step %g lane %d of %d, start step %d pitch %d" % (what, w, h, nscales, scale_step, i, n, step, pitch)
        if variant == "strict":
            want = T.tvl1_init_pyramid(init, lv, scale_step)
            for c in (0, 1):
                for s in range(len(lv)):
                    _bits_equal(got[c][s], want[c][s], "%s: u%d level %d" % (tag, c + 1, s))
            continue
        for c in (0, 1):
            _bits_equal(got[c][0], init[..., c], "%s: u%d level 0" % (tag, c + 1))
            for s in range(1, len(lv)):
                ref = t64.upsample(got[c][s - 1], lv[s][0], lv[s][1], finv, finv, F(scale_step))
                _within(got[c][s], ref, "%s: u%d level %d" % (tag, c + 1, s))


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("shape", FRAMES, ids=["%dx%d" % s for s in FRAMES])
def test_tvl1_start_pyramid_frames(oracle, variant, shape):
    w, h = shape
    e = _handle("tvl1", variant, _size_for(w, h))
    nl = 1 if w * h >= 1920 * 1080 else (2 if w * h >= 1280 * 720 else 3)
    for j, (step, pitch) in enumerate(layouts(w)):
        if w * h > 1920 * 1080 and j % 3 == 0:  # 4K: the padded layouts only (the float64 bound's cost)
            continue
        kind = KINDS[j]
        starts = [start(kind, w, h, 100 * j + i) for i in range(nl)]
        tvl1_case(oracle, e, variant, w, h, 5, 0.8, starts, step, pitch, kind)
    if w * h <= 340 * 256:
        for nscales, scale_step in TVL1_PARAMS:
            tvl1_case(oracle, e, variant, w, h, nscales, scale_step, [start("smooth", w, h, 7 + i) for i in range(nl)], 2, 0, "smooth")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("params", TVL1_PARAMS, ids=["nscales%d-step%g" % p for p in TVL1_PARAMS])
def test_tvl1_start_pyramid_parameters(oracle, variant, params):
    """the CPU pyramid tests' frames and parameters, every start layout and content"""
    nscales, scale_step = params
    e = _handle("tvl1", variant, SMALL)
    for k, (w, h) in enumerate(sorted({(w, h) for w, h, _, _ in PYRAMIDS})):
        for j, (step, pitch) in enumerate(layouts(w)):
            kind = KINDS[(j + k) % 4]
            tvl1_case(oracle, e, variant, w, h, nscales, scale_step, [start(kind, w, h, 10 * k + j + 40 * i) for i in range(3)], step,
                      pitch, kind)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("group", list(GROUPS))
def test_tvl1_start_pyramid_geometry(oracle, variant, group):
    """tiny frames, small planes, strips and the level cuts: one level below 20 px, every layout and content in turn"""
    for k, (w, h) in enumerate(GROUPS[group]):
        e = _handle("tvl1", variant, _size_for(w, h))
        step, pitch = layouts(w)[k % 4]
        kind = KINDS[(k // 4) % 4]
        nscales, scale_step = (5, 0.8) if k % 3 else TVL1_PARAMS[(k // 3) % len(TVL1_PARAMS)]
        n = 1 if w * h > 500 * 500 else 1 + 2 * (k % 2)
        tvl1_case(oracle, e, variant, w, h, nscales, scale_step, [start(kind, w, h, k + 50 * i) for i in range(n)], step, pitch, kind)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("lanes", [1, 3, 16, 17, 40])
def test_tvl1_start_pyramid_lanes(oracle, variant, lanes):
    """more than 16 lanes take several launches of the copy kernel: every lane must still get its own start"""
    e = _handle("tvl1", variant, SMALL)
    for k, (w, h) in enumerate([(340, 256), (131, 97), (33, 17)]):
        for j, (step, pitch) in enumerate(layouts(w)):
            kinds = [KINDS[(i + j + k) % 4] for i in range(lanes)]
            starts = [start(kinds[i], w, h, 1000 * k + 100 * j + i) for i in range(lanes)]
            tvl1_case(oracle, e, variant, w, h, 5, 0.8, starts, step, pitch, "/".join(sorted(set(kinds))))


# ---- Farneback -----------------------------------------------------------------------------------------------------------------
def farn_case(oracle, e, variant, w, h, num_levels, starts, step, pitch, what):
    e.set("num_levels", num_levels)
    p = oracle.farn_params(num_levels=num_levels)
    lv = oracle.farn_levels(w, h, p)
    lw, lh = lv[0][:2]
    n = len(starts)
    x = np.concatenate([s[..., 0] for s in starts])
    y = np.concatenate([s[..., 1] for s in starts])
    outs, _ = e.debug_run_kernel("farn_initial_flow", [x, y], 2, [step, pitch, n], out_shape=(n * lh, lw))
    mul = 1.0
    for _ in range(len(lv) - 1):
        mul *= p.pyr_scale
    for i, init in enumerate(starts):
        tag = "%s %dx%d num_levels %d (coarsest %dx%d) pair %d of %d, start step %d pitch %d" % (what, w, h, num_levels, lw, lh, i, n, step,
                                                                                             pitch)
        got = [o.reshape(n, lh, lw)[i] for o in outs]
        if variant == "strict":
            want = R.farn_start(init, p)
            for c in (0, 1):
                _bits_equal(got[c], want[c], "%s: f%s" % (tag, "xy"[c]))
        else:
            refs = f64.level_start(init[..., 0], init[..., 1], lw, lh, mul)
            for c in (0, 1):
                _within(got[c], refs[c], "%s: f%s" % (tag, "xy"[c]))


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("shape", FRAMES, ids=["%dx%d" % s for s in FRAMES])
def test_farn_start_frames(oracle, variant, shape):
    w, h = shape
    e = _handle("farn", variant, _size_for(w, h))
    n = 1 if w * h >= 1920 * 1080 else 3
    for j, (step, pitch) in enumerate(layouts(w)):
        # 1080p and up: one num_levels per layout (the float64 bound at full resolution is the cost)
        for num_levels in (FARN_LEVELS[j:j + 1] if n == 1 else FARN_LEVELS):
            kind = KINDS[(j + num_levels) % 4]
            farn_case(oracle, e, variant, w, h, num_levels, [start(kind, w, h, 100 * j + 10 * num_levels + i) for i in range(n)], step, pitch,
                      kind)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("group", list(GROUPS))
def test_farn_start_geometry(oracle, variant, group):
    for k, (w, h) in enumerate(GROUPS[group]):
        e = _handle("farn", variant, _size_for(w, h))
        step, pitch = layouts(w)[k % 4]
        kind = KINDS[(k // 4) % 4]
        n = 1 if w * h > 500 * 500 else [1, 3, 8][k % 3]
        farn_case(oracle, e, variant, w, h, FARN_LEVELS[(k // 2) % 4], [start(kind, w, h, k + 50 * i) for i in range(n)], step, pitch, kind)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("pairs", [1, 3, 8])
def test_farn_start_pairs(oracle, variant, pairs):
    e = _handle("farn", variant, SMALL)
    for k, (w, h) in enumerate([(340, 256), (131, 97), (64, 63)]):
        for j, (step, pitch) in enumerate(layouts(w)):
            for num_levels in FARN_LEVELS:
                kinds = [KINDS[(i + j + k) % 4] for i in range(pairs)]
                starts = [start(kinds[i], w, h, 1000 * k + 100 * j + 10 * num_levels + i) for i in range(pairs)]
                farn_case(oracle, e, variant, w, h, num_levels, starts, step, pitch, "/".join(sorted(set(kinds))))
