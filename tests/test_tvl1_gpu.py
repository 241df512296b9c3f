"""GPU parity: CUDA TV-L1 (through the C ABI) vs the CPU oracle on the same seeded inputs.

Tolerance (north_star): average end-point error <= 0.01 px for the default (fast-math-like) build.
The strict build (IEEE, no FMA) performs the oracle's fp32 operations in the oracle's order: its flows and iteration
schedules must equal the oracle's bit for bit.  Only the convergence sum is added in another order; a pair whose result
differs where a check lies within that summation bound of epsilon^2 * pixels is reported as borderline (tests/tvl1_pin.py).
"""
import numpy as np
import pytest

import tvl1_pin as pin
from denseflow_b200 import synth

pytestmark = pytest.mark.gpu

AEE_TOL = 0.01  # px, BASELINE.json north_star
import os
FUSED = [0] if os.environ.get("DFB_SKIP_FUSED") else [0, 1]


def _engine(variant="default", w=256, h=256, **params):
    import denseflow_b200 as d
    e = d.OpticalFlowDual_TVL1.create(0, w, h, variant)
    for k, v in params.items():
        e.set(k, v)
    return e


@pytest.mark.parametrize("fused", FUSED)
@pytest.mark.parametrize("variant", ["strict", "default"])
def test_pair256_matches_oracle(oracle, pair256, variant, fused):
    a, b, gt = pair256
    ref, ref_log, errs = oracle.tvl1_calc(a, b, return_iters=True, return_errors=True)
    e = _engine(variant, fused=fused)
    flow = e.calc(a, b)
    iters, sizes = e.tvl1_stats()
    aee = synth.aee(flow, ref)
    print(variant, "fused", fused, "AEE vs oracle", aee, "max", np.abs(flow - ref).max(), "iters", iters.sum(), ref_log.sum())
    assert sizes == oracle.tvl1_level_sizes(256, 256)
    assert aee <= AEE_TOL
    assert np.isfinite(flow).all()
    assert np.array_equal(e.tvl1_pair_stats(0), iters)
    # sanity vs analytic ground truth (not a parity pin): same ballpark as the oracle
    assert synth.aee(flow, gt) < 0.12
    # executed iteration schedule per (scale, warp): the strict build shares every formula with the oracle, so every
    # convergence decision must come out the same; the default (fast-math-like) build may flip a borderline check
    if variant == "strict":
        pin.finish([pin.check(oracle, a, b, flow, iters, "256x256 fused %d" % fused, oracle_out=(ref, ref_log, errs))])
    else:
        assert abs(int(iters.sum()) - int(ref_log.sum())) <= 0.05 * ref_log.sum()


@pytest.mark.parametrize("fused", FUSED)
def test_iteration_cap_pair(oracle, fused):
    """Independent textures never converge: every (scale, warp) runs into the iteration cap.  The cap is
    lowered to 40 (2 scales x 2 warps) so fp32 chaos cannot build up and the comparison stays tight."""
    a, b = synth.noise_pair(128, 160, 7)
    prm = oracle.tvl1_params(iterations=40, nscales=2, warps=2)
    ref, ref_log = oracle.tvl1_calc(a, b, prm, return_iters=True)
    e = _engine("strict", 160, 128, fused=fused, iterations=40, nscales=2, warps=2)
    flow = e.calc(a, b)
    iters, _ = e.tvl1_stats()
    print("cap pair iters", iters.tolist(), ref_log.tolist())
    assert (iters == 40).all() and (ref_log == 40).all()
    assert np.isfinite(flow).all()
    assert pin.check(oracle, a, b, flow, iters, "cap pair", prm) is None  # the cap decides every check: never borderline
    # full default run: the 300 cap is reached and the result stays finite
    e2 = _engine("default", 160, 128, fused=fused)
    f2 = e2.calc(a, b)
    it2, _ = e2.tvl1_stats()
    assert it2.max() == 300 and np.isfinite(f2).all()


@pytest.mark.parametrize("fused", FUSED)
@pytest.mark.parametrize("shape", [(64, 64), (97, 131), (40, 333), (270, 480)])
def test_odd_sizes(oracle, shape, fused):
    h, w = shape
    a, b, _ = synth.pair(h, w, 3)
    ref = oracle.tvl1_calc(a, b)
    e = _engine("default", w, h, fused=fused)
    flow = e.calc(a, b)
    aee = synth.aee(flow, ref)
    print(shape, "AEE", aee)
    assert aee <= AEE_TOL


def test_small_frame_drops_levels(oracle):
    """A level with cols<16 or rows<16 is dropped (SURVEY A.1)."""
    a, b, _ = synth.pair(24, 40, 5)
    assert len(oracle.tvl1_level_sizes(40, 24)) < 5
    ref = oracle.tvl1_calc(a, b)
    flow = _engine("default", 40, 24).calc(a, b)
    assert synth.aee(flow, ref) <= AEE_TOL


def test_identical_frames_give_zero_flow():
    a, _, _ = synth.pair(128, 128, 1)
    flow = _engine("default", 128, 128).calc(a, a)
    assert np.abs(flow).max() < 1e-3


def test_batch_matches_single_pairs(oracle):
    fr = synth.stream(120, 160, 6, seed=11)
    e = _engine("default", 160, 120)
    flows = e.calc_batch(list(fr), step=1)
    assert flows.shape == (5, 120, 160, 2)
    for i in range(5):
        single = e.calc(fr[i], fr[i + 1])
        assert np.array_equal(single, flows[i])
    assert synth.aee(flows[2], oracle.tvl1_calc(fr[2], fr[3])) <= AEE_TOL
    # negative and larger steps: pair selection of src/denseflow_gpu.cpp:315-316
    fm = e.calc_batch(list(fr), step=-2)
    assert fm.shape == (4, 120, 160, 2)
    assert np.array_equal(fm[1], e.calc(fr[3], fr[1]))
    assert e.calc_batch(list(fr[:2]), step=3).shape[0] == 0


def test_batch_quantised_is_bit_exact(oracle):
    fr = synth.stream(96, 128, 4, seed=12)
    e = _engine("default", 128, 96)
    flows = e.calc_batch(list(fr), step=1)
    qx, qy = e.calc_batch(list(fr), step=1, bound=20)
    for i in range(3):
        ox, oy = oracle.quantise(flows[i], 20)
        assert np.array_equal(qx[i], ox) and np.array_equal(qy[i], oy)


def test_device_path_matches_host_path():
    import torch
    a, b, _ = synth.pair(128, 192, 2)
    e = _engine("default", 192, 128)
    host = e.calc(a, b)
    dev = e.calc(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(host, dev.cpu().numpy())


def test_errors_follow_reference():
    import denseflow_b200 as d
    with pytest.raises(RuntimeError, match="unknown optical algorithm"):
        d.create("lk")
    with pytest.raises(RuntimeError, match="NV hardware flow not enabled"):
        d.create("nv")
    e = _engine("default", 64, 64)
    with pytest.raises(RuntimeError, match="exceeds"):
        e.calc(np.zeros((65, 64), np.uint8), np.zeros((65, 64), np.uint8))


def test_fused_schedule_is_deterministic_and_lane_invariant():
    """Race detector for the persistent kernel: neighbour-warp progress flags, per-warp tile hand-over, grid barriers,
    lanes.  The same batch must come out bit-identical for every lane count, for TMA vs LDG staging, for every k, run to
    run (the repeated entry), and equal to the unfused schedule."""
    fr = synth.stream(360, 640, 9, seed=31)
    ref = None
    for lanes, k, tma in [(1, 8, 0), (1, 8, 1), (2, 8, 1), (4, 8, 0), (8, 8, 1), (8, 8, 1), (3, 5, 1), (0, 3, 1), (0, 1, 1), (0, 2, 0)]:
        e = _engine("default", 640, 360, lanes=lanes, fused_k=k, use_tma=tma)
        out = e.calc_batch(list(fr), step=1)
        if ref is None:
            ref = out
        assert np.array_equal(out, ref), (lanes, k, tma)
    unfused = _engine("default", 640, 360, fused=0).calc_batch(list(fr[:3]), step=1)
    assert np.array_equal(unfused, ref[:2])


def test_one_handle_many_sizes(oracle):
    """A handle created for a maximum size serves any smaller frame (the reference re-creates the algorithm object per
    batch; here the workspace, pyramid slots and TMA descriptors are re-targeted when the geometry changes)."""
    e = _engine("default", 320, 240)
    for (h, w, seed) in [(240, 320, 1), (96, 128, 2), (240, 320, 1), (57, 311, 3), (240, 33, 4)]:
        a, b, _ = synth.pair(h, w, seed)
        ref = oracle.tvl1_calc(a, b)
        assert synth.aee(e.calc(a, b), ref) <= AEE_TOL, (h, w)
    # batches of different sizes back to back, more pairs than lanes
    fr = synth.stream(120, 160, 20, seed=5)
    flows = e.calc_batch(list(fr), step=1)
    assert flows.shape == (19, 120, 160, 2)
    assert synth.aee(flows[18], oracle.tvl1_calc(fr[18], fr[19])) <= AEE_TOL
    assert np.array_equal(flows[7], e.calc(fr[7], fr[8]))


def test_degenerate_batches():
    e = _engine("default", 64, 64)
    fr = [np.zeros((64, 64), np.uint8)] * 3
    assert e.calc_batch(fr[:1], step=1).shape[0] == 0       # one frame: no pair (M = max(N - |step|, 0))
    assert e.calc_batch(fr, step=5).shape[0] == 0           # |step| >= N
    z = e.calc_batch(fr, step=-1)                           # constant frames: exactly zero flow
    assert z.shape == (2, 64, 64, 2) and not z.any()
    with pytest.raises(RuntimeError):
        e.calc_batch(fr, step=0)                            # step 0 is the frame-extraction mode, not a flow request


# ---- the configurations the headline numbers are quoted on (BASELINE.json configs[2] and [4]) ------------------------
def _check_batch_against_oracle(oracle, fr, w, h, variant, pairs_to_check, tol):
    e = _engine(variant, w, h)
    flows = e.calc_batch(list(fr), step=1)
    lanes = int(e.get("lanes")) or None
    worst = 0.0
    notes = []
    for j in pairs_to_check:
        ref, ref_log, errs = oracle.tvl1_calc(fr[j], fr[j + 1], return_iters=True, return_errors=True)
        aee = synth.aee(flows[j], ref)
        worst = max(worst, aee)
        log = e.tvl1_pair_stats(j)
        print("%dx%d %s pair %d: AEE %.3e px, iterations %d (oracle %d)" % (w, h, variant, j, aee, log.sum(), ref_log.sum()))
        assert np.isfinite(flows[j]).all()
        assert aee <= tol, (j, aee)
        if variant == "strict":
            notes.append(pin.check(oracle, fr[j], fr[j + 1], flows[j], log, "%dx%d pair %d" % (w, h, j), oracle_out=(ref, ref_log, errs)))
        else:
            assert abs(int(log.sum()) - int(ref_log.sum())) <= 0.05 * ref_log.sum()
    pin.finish(notes)
    return worst


@pytest.mark.parametrize("variant", ["strict", "default"])
def test_1080p_batch_matches_oracle(oracle, variant):
    """BASELINE.json configs[2]: 1920x1080, nine frames = eight pairs, spread over launches of the automatically chosen
    lane count (which depends on the GPU's SM count); every flow is compared with the oracle, and for the strict build the
    executed iterations per (scale, warp) must be identical."""
    oracle.lib().orc_set_num_threads(min(16, oracle.usable_cores()))
    fr = synth.stream(1080, 1920, 9, seed=1)
    pairs = range(8) if variant == "strict" else (0, 6, 7)  # default build: the first pair and the last two
    _check_batch_against_oracle(oracle, fr, 1920, 1080, variant, pairs, 1e-3 if variant == "strict" else AEE_TOL)
    oracle.lib().orc_set_num_threads(min(8, oracle.usable_cores()))


@pytest.mark.parametrize("variant", ["strict", "default"])
def test_340x256_clip_matches_oracle(oracle, variant):
    """BASELINE.json configs[4]: one 340x256 x 64-frame clip = 63 pairs, several lanes per launch."""
    fr = synth.stream(256, 340, 64, seed=100)
    pairs = range(63) if variant == "strict" else range(0, 63, 4)
    _check_batch_against_oracle(oracle, fr, 340, 256, variant, pairs, 1e-3 if variant == "strict" else AEE_TOL)
