"""-st=h5 payloads on the GPU: the engines' planar merge epilogue (fused and unfused TV-L1, Farneback) writes each pair's flow as
two float planes, and every planar entry point gives bit for bit the x and y channels of the float2 path (calc_batch)."""
import numpy as np
import pytest

import denseflow_b200 as d
from denseflow_b200 import synth

pytestmark = pytest.mark.gpu


def _engine(alg, w, h, variant="default", **params):
    e = d.create(alg, 0, w, h, variant=variant)
    for k, v in params.items():
        e.set(k, v)
    return e


def _split(flows):
    return np.ascontiguousarray(np.moveaxis(flows, -1, 1))


def _pinned(shape):
    import torch
    return torch.empty(shape, dtype=torch.float32, pin_memory=True).numpy()


def _assert_planes(planes, flows):
    want = _split(flows)
    assert planes.shape == want.shape and planes.dtype == np.float32
    assert planes.tobytes() == want.tobytes()


CASES = [
    # (algorithm, w, h, n_frames, step, params)
    ("tvl1", 340, 256, 6, 1, {}),
    ("tvl1", 340, 256, 7, -3, {}),
    ("tvl1", 340, 256, 5, 3, {"fused": 0}),
    ("tvl1", 340, 256, 4, -1, {"fused": 0, "median_filtering": 5, "median_interval": 7}),
    ("tvl1", 340, 256, 6, 1, {"median_filtering": 3, "median_interval": 30}),
    ("tvl1", 340, 256, 6, 1, {"lanes": 2, "use_tma": 0, "fused_k": 3}),
    ("tvl1", 97, 131, 3, 1, {}),
    ("tvl1", 1080, 7, 3, -1, {}),
    ("tvl1", 1, 1, 2, 1, {}),
    ("farn", 340, 256, 6, 1, {}),
    ("farn", 340, 256, 12, -3, {}),
    ("farn", 97, 131, 3, 1, {}),
    ("farn", 1080, 7, 4, 3, {}),
]


@pytest.mark.parametrize("variant", ["default", "strict"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_planes_equal_the_float2_path(case, variant):
    alg, w, h, n, step, params = CASES[case]
    fr = synth.stream(h, w, n, seed=case)
    e = _engine(alg, w, h, variant, **params)
    flows = e.calc_batch(list(fr), step=step)
    _assert_planes(e.calc_batch_planes(list(fr), step=step), flows)
    _assert_planes(e.calc_batch_planes(list(fr), step=step, out=_pinned(flows.shape[:1] + (2, h, w))), flows)
    import torch
    dev = e.calc_batch_device_planes(torch.from_numpy(fr).cuda(), step=step)
    torch.cuda.synchronize()
    _assert_planes(dev.cpu().numpy(), flows)
    e.release()


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("n", [0, 1, 3, 4, 20])
def test_frame_counts_and_groups(alg, n):
    """0 and 1 frames, |step| frames (no pair), and more pairs than one group holds"""
    w, h = 64, 48
    fr = synth.stream(h, w, max(n, 1), seed=n)[:n]
    e = _engine(alg, w, h, lanes=2) if alg == "tvl1" else _engine(alg, w, h)
    for step in (3, -1):
        flows = e.calc_batch(list(fr), step=step) if n else np.empty((0, h, w, 2), np.float32)
        planes = e.calc_batch_planes(list(fr), step=step)
        if n:
            _assert_planes(planes, flows)
        else:
            assert planes.shape[0] == 0
    e.release()


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_1080p(alg):
    fr = synth.stream(1080, 1920, 3, seed=5)
    e = _engine(alg, 1920, 1080)
    flows = e.calc_batch(list(fr), step=1)
    _assert_planes(e.calc_batch_planes(list(fr), step=1, out=_pinned((2, 2, 1080, 1920))), flows)
    e.release()


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_strict_planes_against_the_oracle(oracle, alg):
    a, b, _ = synth.pair(128, 160, 3)
    e = _engine(alg, 160, 128, "strict")
    p = e.calc_batch_planes([a, b])[0]
    ref = oracle.tvl1_calc(a, b) if alg == "tvl1" else oracle.farn_calc(a, b)
    assert synth.aee(np.stack([p[0], p[1]], -1), ref) <= (1e-3 if alg == "tvl1" else 1e-4)
    e.release()


def _bgr_clip(n, h, w, seed):
    g = synth.stream(h, w, n, seed)
    rng = np.random.default_rng(seed)
    return [np.ascontiguousarray(np.stack([f, np.roll(f, 3, 1), (f // 2 + rng.integers(0, 64, f.shape)).astype(np.uint8)], -1))
            for f in g]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("new_size", [None, (171, 128)])
def test_colour_chains(alg, new_size):
    import cv2
    frames = _bgr_clip(6, 256, 340, 11)
    e = _engine(alg, 340, 256)
    gray = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in frames]
    if new_size:
        gray = [cv2.resize(g, new_size) for g in gray]
    for step in (1, -3):
        want = e.calc_batch_planes(gray, step=step)
        got = e.process_bgr_batch_planes(frames, step=step, new_size=new_size)
        assert got.tobytes() == want.tobytes()
        jpegs = [cv2.imencode(".jpg", f)[1].tobytes() for f in frames]
        dec = [cv2.cvtColor(cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY) for j in jpegs]
        if new_size:
            dec = [cv2.resize(g, new_size) for g in dec]
        assert e.process_jpeg_batch_planes(jpegs, step=step, new_size=new_size).tobytes() == e.calc_batch_planes(dec, step=step).tobytes()
    e.release()


def test_planes_refusals():
    import ctypes as C
    e = _engine("tvl1", 64, 48)
    fr = synth.stream(48, 64, 3, 0)
    with pytest.raises(RuntimeError, match="step must be non-zero"):
        e.calc_batch_planes(list(fr), step=0)
    L = e._L
    fp = (C.c_void_p * 3)(*[f.ctypes.data for f in fr])
    assert L.dfb_calc_batch_host_planes(e._h, fp, 3, 1, 64, 48, None, None) == -1
    assert b"fx/fy is null" in L.dfb_last_error(e._h)
    e.release()
