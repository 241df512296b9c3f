"""GPU imencode(".png") (denseflow_b200/csrc/png_encode.cu) byte-identical to the restatement (tests/png_restate.py, pinned to
cv2 and to golden bytes in tests/test_png_encode_cpu.py), in both builds, and the -st=png batch call against the flows the
same handle computes."""
import ctypes as C
import os

import numpy as np
import pytest

import geometry_cases as G
import inflate_trace as T
import png_cases as PC
import png_restate as P
from denseflow_b200 import _lib, synth
from oracle import cv_restate as R

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png_imencode_cases.npz")

_handles = {}


def handle(alg="tvl1", variant="default", size=(3840, 2160)):
    import denseflow_b200 as d
    key = (alg, variant, size)
    if key not in _handles:
        _handles[key] = d.create(alg, 0, size[0], size[1], variant=variant)
    return _handles[key]


def _check(e, img, **kw):
    import torch
    import cv2
    got = e.encode_png_bgr_device(torch.from_numpy(np.ascontiguousarray(img)).cuda(), **kw)
    want = P.encode(img)
    assert got == want, (img.shape, len(got), len(want), T.first_difference(P.idat_stream(got), P.idat_stream(want)))
    assert np.array_equal(cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_COLOR), img)
    return got


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_tiny_sizes(variant):
    e = handle(variant=variant)
    for w, h in G.TINY:
        for kind in ("noise", "constant", "mixed"):
            _check(e, PC.image(kind, h, w))


@pytest.mark.parametrize("variant", ["default", "strict"])
@pytest.mark.parametrize("shape", PC.BLOCK_EDGE_SIZES + [(130, 42), (128, 42)])
def test_deflate_block_edges(shape, variant):
    e = handle(variant=variant)
    _check(e, PC.literal_noise(*shape))
    for kind in PC.CONTENTS:
        _check(e, PC.image(kind, *shape))


@pytest.mark.parametrize("wh", G.STRIPS + [(340, 256), (1280, 720), (1920, 1080), (3840, 2160)])
def test_frame_sizes(wh):
    w, h = wh
    e = handle()
    for kind in PC.CONTENTS:
        _check(e, PC.image(kind, h, w))
    _check(e, PC.ramp(h, w))


@pytest.mark.parametrize("n", [3, 4, 258, 259, 260, 261, 517])
def test_runs(n):
    _check(handle(), PC.run_image(n))


def test_golden_bytes():
    import torch
    g = np.load(GOLDEN)
    e = handle()
    for i in range(sum(1 for k in g.files if k.startswith("img"))):
        img = g["img%d" % i]
        assert e.encode_png_bgr_device(torch.from_numpy(img).cuda()) == g["png%d" % i].tobytes(), i


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("variant", ["default", "strict"])
def test_packed_engine_flows(alg, variant):
    """The images -st=png encodes: convertFlowToPngImage of engine flows, on either kind of handle."""
    e = handle(alg, variant, (340, 256))
    for h, w in [(256, 340), (96, 128), (5, 7)]:
        a, b, _ = synth.pair(h, w, 3)
        flow = e.calc(a, b)
        img, _, _ = R.flow_to_png_image(flow)
        _check(e, img)


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_pitched_offset_source_on_a_stream(offset):
    import torch
    e = handle()
    h, w = 37, 53
    img = PC.image("smooth", h, w)
    pitch = 3 * w + 29
    buf = torch.zeros(offset + pitch * h, dtype=torch.uint8, device="cuda")
    view = buf[offset:].as_strided((h, w, 3), (pitch, 3, 1))
    view.copy_(torch.from_numpy(img))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = e.encode_png_bgr_device(view)
        got2 = e.encode_png_bgr_device(view)  # two calls in a row
    assert got == got2 == P.encode(img)


def test_too_small_capacity_then_next_call():
    import torch
    e = handle()
    img = PC.image("noise", 20, 30)
    want = P.encode(img)
    dev = torch.from_numpy(img).cuda()
    with pytest.raises(RuntimeError, match="needs %d bytes" % len(want)):
        e.encode_png_bgr_device(dev, capacity=len(want) - 1)
    assert e.encode_png_bgr_device(dev, capacity=len(want)) == want
    assert e.encode_png_bgr_device(dev) == want


def test_argument_checks():
    import torch
    e = handle(size=(64, 48))
    L, hd = e._L, e._h
    img = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")
    out = np.empty(L.dfb_png_max_bytes(8, 8), np.uint8)
    n = C.c_size_t()
    enc = L.dfb_encode_png_bgr_device
    assert enc(hd, None, 24, 8, 8, out.ctypes.data, out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG
    assert enc(hd, img.data_ptr(), 24, 8, 8, None, out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG
    assert enc(hd, img.data_ptr(), 24, 8, 8, out.ctypes.data, out.size, None, None) == _lib.DFB_ERR_INVALID_ARG
    assert enc(hd, img.data_ptr(), 23, 8, 8, out.ctypes.data, out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG
    assert enc(hd, img.data_ptr(), 24, 8, 8, img.data_ptr(), out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG  # device output
    host = np.zeros((8, 8, 3), np.uint8)
    assert enc(hd, host.ctypes.data, 24, 8, 8, out.ctypes.data, out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG  # host input
    big = torch.zeros((49, 8, 3), dtype=torch.uint8, device="cuda")
    assert enc(hd, big.data_ptr(), 24, 8, 49, out.ctypes.data, out.size, C.byref(n), None) == _lib.DFB_ERR_SIZE
    assert enc(None, img.data_ptr(), 24, 8, 8, out.ctypes.data, out.size, C.byref(n), None) == _lib.DFB_ERR_INVALID_ARG
    # the batch call
    frames = [np.zeros((8, 8), np.uint8) for _ in range(3)]
    fp = (C.c_void_p * 3)(*[f.ctypes.data for f in frames])
    bufs = [np.empty(out.size, np.uint8) for _ in range(2)]
    op = (C.c_void_p * 2)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * 2)()
    batch = L.dfb_calc_batch_host_png
    assert batch(hd, fp, 3, 1, 8, 8, None, out.size, lens) == _lib.DFB_ERR_INVALID_ARG
    assert batch(hd, fp, 3, 1, 8, 8, op, out.size, None) == _lib.DFB_ERR_INVALID_ARG
    assert batch(hd, fp, 3, 0, 8, 8, op, out.size, lens) == _lib.DFB_ERR_INVALID_ARG
    dop = (C.c_void_p * 2)(bufs[0].ctypes.data, img.data_ptr())
    assert batch(hd, fp, 3, 1, 8, 8, dop, out.size, lens) == _lib.DFB_ERR_INVALID_ARG
    assert "device pointer" in L.dfb_last_error(hd).decode()
    nop = (C.c_void_p * 2)(bufs[0].ctypes.data, None)
    assert batch(hd, fp, 3, 1, 8, 8, nop, out.size, lens) == _lib.DFB_ERR_INVALID_ARG
    big_frames = [np.zeros((49, 8), np.uint8) for _ in range(3)]
    bfp = (C.c_void_p * 3)(*[f.ctypes.data for f in big_frames])
    assert batch(hd, bfp, 3, 1, 8, 49, op, out.size, lens) == _lib.DFB_ERR_SIZE
    with pytest.raises(RuntimeError, match="too small"):
        _small_batch(e, frames)
    assert e.calc_batch_png(frames) == [P.encode(R.flow_to_png_image(f)[0]) for f in e.calc_batch(frames)]


def _small_batch(e, frames):
    L = e._L
    bufs = [np.empty(64, np.uint8) for _ in range(2)]
    fp = (C.c_void_p * 3)(*[f.ctypes.data for f in frames])
    op = (C.c_void_p * 2)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * 2)()
    e._check(L.dfb_calc_batch_host_png(e._h, fp, 3, 1, 8, 8, op, 64, lens))


def _pinned(n, cap):
    import torch
    return [torch.empty(cap, dtype=torch.uint8, pin_memory=True).numpy() for _ in range(n)]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("step", [1, -1, 3, -3])
@pytest.mark.parametrize("n_frames", [0, 1, 2, 9, 19])
def test_batch_equals_flow_then_encode(alg, step, n_frames):
    e = handle(alg, "default", (96, 64))
    frames = list(synth.stream(64, 96, n_frames, 5)) if n_frames else []
    flows = e.calc_batch(frames, step=step) if n_frames else np.empty((0, 64, 96, 2), np.float32)
    m = max(n_frames - abs(step), 0)
    want = [P.encode(R.flow_to_png_image(flows[j])[0]) for j in range(m)]
    assert e.calc_batch_png(frames, step=step) == want
    if m:
        assert e.calc_batch_png(frames, step=step, out=_pinned(m, e._L.dfb_png_max_bytes(96, 64))) == want
        assert np.array_equal(e.calc_batch(frames, step=step), flows)  # a flow call after a PNG call


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("variant", ["default", "strict"])
def test_batch_over_several_groups(alg, variant):
    """More pairs than one group at 1080p (groups of at most 7 TV-L1 pairs there), pageable and page-locked outputs"""
    e = handle(alg, variant, (1920, 1080))
    frames = list(synth.stream(1080, 1920, 10, 11))
    flows = e.calc_batch(frames)
    want = [P.encode(R.flow_to_png_image(f)[0]) for f in flows]
    assert e.calc_batch_png(frames) == want
    assert e.calc_batch_png(frames, out=_pinned(len(want), e._L.dfb_png_max_bytes(1920, 1080))) == want
    assert np.array_equal(e.calc_batch(frames), flows)
