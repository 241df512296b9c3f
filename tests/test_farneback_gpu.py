"""GPU parity: CUDA Farneback (through the C ABI) vs the CPU oracle (CUDA resize convention), which itself
is pinned to OpenCV's CPU Farneback (tests/test_oracle_cpu.py)."""
import numpy as np
import pytest

from denseflow_b200 import synth

pytestmark = pytest.mark.gpu
AEE_TOL = 0.01


def _engine(w, h, variant="default"):
    import denseflow_b200 as d
    return d.FarnebackOpticalFlow.create(0, w, h, variant)


@pytest.mark.parametrize("variant", ["strict", "default"])
@pytest.mark.parametrize("shape", [(256, 256), (256, 340), (97, 131), (64, 64), (360, 640)])
def test_farneback_matches_oracle(oracle, shape, variant):
    h, w = shape
    a, b, gt = synth.pair(h, w, 0)
    ref = oracle.farn_calc(a, b)
    flow = _engine(w, h, variant).calc(a, b)
    aee = synth.aee(flow, ref)
    print(shape, variant, "AEE vs oracle", aee, "max", np.abs(flow - ref).max())
    assert np.isfinite(flow).all()
    assert aee <= (1e-4 if variant == "strict" else AEE_TOL)
    if min(h, w) >= 128:
        assert synth.aee(flow, gt) < 0.15  # sanity vs analytic flow (CPU Farneback gets 0.04-0.07 px here)


def test_farneback_small_frame_level_cropping(oracle):
    """Fewer than 5 levels when W*0.5^k < 32 (SURVEY B.1)."""
    a, b, _ = synth.pair(96, 160, 2)
    assert len(oracle.farn_levels(160, 96)) == 2  # 160x96 -> 80x48 kept, 40x24 dropped (24 < 32)
    assert len(oracle.farn_levels(80, 48)) == 1
    assert synth.aee(_engine(160, 96).calc(a, b), oracle.farn_calc(a, b)) <= AEE_TOL
    a, b, _ = synth.pair(48, 80, 2)
    assert synth.aee(_engine(80, 48).calc(a, b), oracle.farn_calc(a, b)) <= AEE_TOL


def test_farneback_batch_and_quantise(oracle):
    fr = synth.stream(120, 160, 5, seed=21)
    e = _engine(160, 120)
    flows = e.calc_batch(list(fr), step=1)
    assert flows.shape == (4, 120, 160, 2)
    for i in range(4):
        assert np.array_equal(flows[i], e.calc(fr[i], fr[i + 1]))
    assert synth.aee(flows[1], oracle.farn_calc(fr[1], fr[2])) <= AEE_TOL
    qx, qy = e.calc_batch(list(fr), step=2, bound=20)
    f2 = e.calc_batch(list(fr), step=2)
    for i in range(3):
        ox, oy = oracle.quantise(f2[i], 20)
        assert np.array_equal(qx[i], ox) and np.array_equal(qy[i], oy)


def test_farneback_720p_config(oracle):
    """BASELINE.json configs[3] size."""
    fr = synth.stream(720, 1280, 2, seed=2)
    ref = oracle.farn_calc(fr[0], fr[1])
    flow = _engine(1280, 720).calc(fr[0], fr[1])
    assert synth.aee(flow, ref) <= AEE_TOL


def test_farneback_1080p_six_levels(oracle):
    """1920x1080 keeps the k = 5 level (60 x 34): smoothSize 79, the widest Gaussian of the path."""
    assert oracle.farn_levels(1920, 1080)[0][:3] == (60, 34, 79)
    fr = synth.stream(1080, 1920, 2, seed=1)
    ref = oracle.farn_calc(fr[0], fr[1])
    flow = _engine(1920, 1080).calc(fr[0], fr[1])
    assert synth.aee(flow, ref) <= AEE_TOL


@pytest.mark.parametrize("shape", [(97, 131), (360, 640), (720, 1280)])
def test_batched_iteration_matches_single_pairs(shape):
    """The persistent iteration kernel walks one tile list over pairs x tile rows x tile columns: every pair of a batched
    7-frame stream equals the same handle's one-pair calc of that pair (a tile list of one pair), bit for bit, at odd sizes
    with partial tiles; and the batch is the same from run to run (stage reuse, mbarrier phases)."""
    h, w = shape
    fr = synth.stream(h, w, 7, seed=40)
    e = _engine(w, h)
    b = e.calc_batch(list(fr), step=1)
    for i in range(len(fr) - 1):
        assert np.array_equal(b[i], e.calc(fr[i], fr[i + 1])), i
    assert np.array_equal(b, e.calc_batch(list(fr), step=1))
