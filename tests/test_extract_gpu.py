"""Frame-extraction mode (`-s=0`) on the GPU: the colour preparation kernel bit for bit against the restatement of
cv::resize + libjpeg's YCbCr 4:2:0 sampling, nvJPEG's colour JPEGs against imencode's round trip, the batch entry point
against the single-frame one, and the argument checks."""
import ctypes as C

import numpy as np
import pytest

import geometry_cases as gc
import ycc_restate as Y
from denseflow_b200 import _lib, synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def eng():
    import denseflow_b200 as d
    return d.FarnebackOpticalFlow.create(0, 2048, 2048)


def _colour(gray, seed=0):
    """colour frames whose three channels differ (as tests/test_pipeline_gpu.py builds them)"""
    rng = np.random.default_rng(seed)
    return [np.stack([np.roll(g, 3, 1), g, 255 - np.roll(g, 5, 0)], -1).astype(np.uint8) ^ rng.integers(0, 4, g.shape + (3,), dtype=np.uint8)
            for g in gray]


def _ref(bgr, dst):
    h, w = bgr.shape[:2]
    return Y.bgr_to_ycc420(cv2.resize(bgr, dst) if dst and tuple(dst) != (w, h) else bgr)


def _check_planes(e, bgr_dev, bgr, dst, what=""):
    import torch
    got = e.bgr_to_ycc420_device(bgr_dev, dst)
    torch.cuda.synchronize()
    for g, r, name in zip(got, _ref(bgr, dst), "y cb cr".split()):
        assert np.array_equal(g.cpu().numpy(), r), (what, name, bgr.shape, dst)


@pytest.mark.parametrize("src, dst", [((1920, 1080), None), ((1920, 1080), (340, 256)), ((1920, 1080), (960, 540)), ((1920, 1080), (455, 256)),
                                      ((320, 240), (640, 480)), ((37, 23), (75, 47)), ((641, 479), (1, 1)), ((100, 3), (7, 201))])
def test_ycc420_kernel_bit_exact(eng, src, dst):
    import torch
    (sw, sh) = src
    bgr = np.random.default_rng(sw + sh).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    _check_planes(eng, torch.from_numpy(bgr).cuda(), bgr, dst)


def test_ycc420_kernel_tiny_destinations(eng):
    """every dw, dh in 1..8 and 15 / 16 / 17, resized from 37 x 23 and taken as they are"""
    import torch
    rng = np.random.default_rng(3)
    src = rng.integers(0, 256, (23, 37, 3), dtype=np.uint8)
    dev = torch.from_numpy(src).cuda()
    sizes = list(range(1, 9)) + [15, 16, 17]
    for dw in sizes:
        for dh in sizes:
            _check_planes(eng, dev, src, (dw, dh), "resize")
            own = rng.integers(0, 256, (dh, dw, 3), dtype=np.uint8)
            _check_planes(eng, torch.from_numpy(own).cuda(), own, None, "as is")


@pytest.mark.parametrize("src, dst", [((1, 1920), (1, 960)), ((1920, 1), (960, 1)), ((7, 1080), (3, 541)), ((1080, 7), (541, 3)),
                                      ((1, 1920), None), ((1920, 1), None), ((7, 1080), None), ((2000, 13), (2001, 1)), ((1, 1), (5, 3))])
def test_ycc420_kernel_thin_strips(eng, src, dst):
    import torch
    (sw, sh) = src
    bgr = np.random.default_rng(sw * 7 + sh).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    _check_planes(eng, torch.from_numpy(bgr).cuda(), bgr, dst)


def _offset_view(img, off, extra):
    """img copied into a device buffer whose rows are `extra` bytes longer than the image and whose base is `off` bytes
    past an aligned address"""
    import torch
    h, row = img.shape[0], img[0].size
    pitch = row + extra
    buf = torch.zeros(h * pitch + off, dtype=torch.uint8, device="cuda")
    v = torch.as_strided(buf, img.shape, (pitch, 3, 1), off)
    v.copy_(torch.from_numpy(img))
    assert v.data_ptr() % 4 == off % 4 and v.stride(0) == pitch
    return v


@pytest.mark.parametrize("off, extra", [(1, 3), (2, 5), (3, 64)])
def test_ycc420_kernel_from_pitched_offset_sources(eng, off, extra):
    rng = np.random.default_rng(off)
    for (sw, sh), dst in [((131, 97), None), ((131, 97), (64, 48)), ((7, 5), (17, 15)), ((1, 1), None), ((33, 17), (16, 9))]:
        bgr = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        _check_planes(eng, _offset_view(bgr, off, extra), bgr, dst, (off, extra))


def test_ycc420_kernel_on_its_own_stream(eng):
    import torch
    bgr = np.random.default_rng(9).integers(0, 256, (480, 640, 3), dtype=np.uint8)
    dev = torch.from_numpy(bgr).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = eng.bgr_to_ycc420_device(dev, (340, 256))
    s.synchronize()
    for g, r in zip(got, _ref(bgr, (340, 256))):
        assert np.array_equal(g.cpu().numpy(), r)


def test_ycc420_kernel_on_every_bgr_triple():
    """all 2^24 BGR triples as one 4096 x 4096 frame, no resize: Y per pixel, Cb / Cr per 2 x 2 block"""
    import torch
    import denseflow_b200 as d
    e = d.FarnebackOpticalFlow.create(0, 4096, 4096)
    i = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    y, cb, cr = e.bgr_to_ycc420_device(torch.from_numpy(bgr).cuda())
    torch.cuda.synchronize()
    for g, r in zip((y, cb, cr), Y.bgr_to_ycc420(bgr)):
        assert np.array_equal(g.cpu().numpy(), r)


# ---- nvJPEG colour encode ----------------------------------------------------------------------------------------
def _frames(w, h, n, seed=41):
    return _colour(synth.stream(h, w, n, seed=seed), seed)


# decoded error against the resized frame, as measured for imencode's own round trip, plus these margins: a regression
# guard over the residuals measured on an H100 80GB HBM3 at 700 W (max error equal to imencode's at every size below, mean
# error at most 0.028 above it)
MAX_MARGIN, MEAN_MARGIN = 2, 0.1


@pytest.mark.parametrize("src, dst", [((1920, 1080), (340, 256)), ((1920, 1080), None), ((640, 480), (341, 255)), ((256, 192), (17, 9)),
                                      ((256, 192), (1, 1)), ((256, 192), (33, 2)), ((257, 193), None)])
def test_encode_decodes_like_opencv(eng, src, dst):
    import torch
    (sw, sh) = src
    bgr = _frames(sw, sh, 1)[0]
    resized = cv2.resize(bgr, dst) if dst else bgr
    dw, dh = dst if dst else src
    jpg = eng.encode_jpeg_bgr_device(torch.from_numpy(bgr).cuda(), dst)
    assert jpg[:2] == b"\xff\xd8" and jpg[-2:] == b"\xff\xd9"
    dec = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_UNCHANGED)
    assert dec.shape == (dh, dw, 3) and dec.dtype == np.uint8
    ok, ref = cv2.imencode(".jpg", resized)  # OpenCV defaults: quality 95, 4:2:0
    ref_dec = cv2.imdecode(ref, cv2.IMREAD_UNCHANGED)
    err = np.abs(dec.astype(int) - resized.astype(int))
    ref_err = np.abs(ref_dec.astype(int) - resized.astype(int))
    print("extract %s->%s nvjpeg bytes %d opencv bytes %d max err %d (opencv %d) mean %.4f (opencv %.4f)"
          % (src, (dw, dh), len(jpg), len(ref), err.max(), ref_err.max(), err.mean(), ref_err.mean()))
    assert err.max() <= ref_err.max() + MAX_MARGIN and err.mean() <= ref_err.mean() + MEAN_MARGIN
    if dw * dh >= 64 * 64:  # headers dominate tiny images
        assert 0.5 < len(jpg) / len(ref) < 2.0


def test_encode_quality_is_honoured(eng):
    import torch
    bgr = torch.from_numpy(_frames(340, 256, 1)[0]).cuda()
    sizes = [len(eng.encode_jpeg_bgr_device(bgr, None, q)) for q in (50, 75, 95, 100)]
    assert sizes == sorted(sizes) and sizes[0] < sizes[-1]


# ---- the batch entry point -----------------------------------------------------------------------------------------
def _pinned(frames):
    import torch
    out = []
    for f in frames:
        t = torch.empty(f.shape, dtype=torch.uint8, pin_memory=True)
        t.numpy()[...] = f
        out.append(t.numpy())
    return out


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("n, dst", [(0, None), (1, (340, 256)), (9, None), (9, (171, 129)), (19, (340, 256))])
def test_extract_frames_equals_single_frame_encodes(alg, pinned, n, dst):
    import torch
    import denseflow_b200 as d
    e = d.create(alg, 0, 640, 480)
    frames = _frames(480, 360, max(n, 1))[:n]
    if pinned:
        frames = _pinned(frames)
    before = e.counters()
    out = e.extract_frames(frames, dst)
    after = e.counters()
    assert len(out) == n
    assert after["kernel_launches"] - before["kernel_launches"] == n
    assert after["h2d_bytes"] - before["h2d_bytes"] == n * 480 * 360 * 3
    assert after["d2h_bytes"] - before["d2h_bytes"] == sum(len(j) for j in out)
    assert after["pairs"] == before["pairs"]
    for f, jpg in zip(frames, out):
        assert jpg == e.encode_jpeg_bgr_device(torch.from_numpy(np.array(f)).cuda(), dst)


def test_extract_frames_leaves_the_flow_alone():
    """a flow call, frame extraction and flow again on one handle: the flow is unchanged"""
    import denseflow_b200 as d
    for alg in ("tvl1", "farn"):
        e = d.create(alg, 0, 256, 192)
        a, b, _ = synth.pair(192, 256, 3)
        first = e.calc(a, b).copy()
        q_first = e.calc_batch([a, b, a], step=1, bound=20)
        e.extract_frames(_frames(256, 192, 10), (128, 96))
        assert np.array_equal(e.calc(a, b), first)
        q = e.calc_batch([a, b, a], step=1, bound=20)
        assert all(np.array_equal(x, y) for x, y in zip(q, q_first))


# ---- argument checks -------------------------------------------------------------------------------------------------
def _err(e):
    return e._L.dfb_last_error(e._h).decode()


def test_ycc420_argument_checks():
    import torch
    import denseflow_b200 as d
    e = d.create("farn", 0, 64, 48)
    L, h = e._L, e._h
    bgr = torch.zeros((48, 64, 3), dtype=torch.uint8, device="cuda")
    y = torch.empty((48, 64), dtype=torch.uint8, device="cuda")
    c = torch.empty((24, 32), dtype=torch.uint8, device="cuda")
    host = np.zeros((48, 64, 3), np.uint8)
    ok = (bgr.data_ptr(), 192, 64, 48, 0, 0, y.data_ptr(), 64, c.data_ptr(), c.data_ptr(), 32, None)
    assert L.dfb_bgr_to_ycc420_device(h, *ok) == _lib.DFB_OK
    torch.cuda.synchronize()

    def call(**kw):
        names = "bgr pitch sw sh dw dh y y_pitch cb cr c_pitch stream".split()
        args = dict(zip(names, ok))
        args.update(kw)
        return L.dfb_bgr_to_ycc420_device(h, *[args[k] for k in names])
    for kw in [dict(bgr=None), dict(y=None), dict(cb=None), dict(cr=None), dict(bgr=host.ctypes.data), dict(y=host.ctypes.data),
               dict(sw=0), dict(sh=-1), dict(dw=5), dict(dh=5), dict(dw=-1, dh=-1), dict(pitch=191), dict(y_pitch=63), dict(c_pitch=31),
               dict(dw=9, dh=9, c_pitch=4)]:
        assert call(**kw) == _lib.DFB_ERR_INVALID_ARG, kw
    assert call(sw=65, pitch=195) == _lib.DFB_ERR_SIZE  # no resize: the destination is the 65 x 48 source
    assert "exceeds" in _err(e)
    assert call(dw=64, dh=49) == _lib.DFB_ERR_SIZE
    assert call(dw=128, dh=96, sw=32, sh=24) == _lib.DFB_ERR_SIZE
    assert L.dfb_bgr_to_ycc420_device(None, *ok) == _lib.DFB_ERR_INVALID_ARG


def test_encode_argument_checks_and_capacity():
    import torch
    import denseflow_b200 as d
    e = d.create("tvl1", 0, 64, 48)
    L, h = e._L, e._h
    bgr = torch.from_numpy(_frames(64, 48, 1)[0]).cuda()
    cap = L.dfb_jpeg_max_bytes_bgr(64, 48)
    out = np.empty(cap, np.uint8)
    n = C.c_size_t()
    dev_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    base = [bgr.data_ptr(), 192, 64, 48, 0, 0, 95, out.ctypes.data, cap, C.byref(n), None]
    assert L.dfb_encode_jpeg_bgr_device(h, *base) == _lib.DFB_OK and n.value > 0
    need = n.value
    for i, v in [(6, 0), (6, 101), (0, None), (7, None), (9, None), (0, np.zeros(9216, np.uint8).ctypes.data), (7, dev_out.data_ptr()),
                 (2, 0), (4, 10)]:
        args = list(base)
        args[i] = v
        assert L.dfb_encode_jpeg_bgr_device(h, *args) == _lib.DFB_ERR_INVALID_ARG, (i, v)
    args = list(base)
    args[4:6] = [65, 48]
    assert L.dfb_encode_jpeg_bgr_device(h, *args) == _lib.DFB_ERR_SIZE
    # a capacity one byte short: a clean failure naming the length, and nothing written past the capacity
    guard = np.full(need + 64, 0xA5, np.uint8)
    args = list(base)
    args[7:9] = [guard.ctypes.data, need - 1]
    assert L.dfb_encode_jpeg_bgr_device(h, *args) == _lib.DFB_ERR_INVALID_ARG
    assert "needs %d bytes" % need in _err(e)
    assert (guard[need - 1:] == 0xA5).all()
    # the handle still works
    assert L.dfb_encode_jpeg_bgr_device(h, *base) == _lib.DFB_OK and n.value == need


def test_extract_frames_argument_checks_and_capacity():
    import torch
    import denseflow_b200 as d
    e = d.create("farn", 0, 64, 48)
    L, h = e._L, e._h
    frames = _frames(64, 48, 10)
    cap = L.dfb_jpeg_max_bytes_bgr(64, 48)
    outs = [np.empty(cap, np.uint8) for _ in frames]
    fp = (C.c_void_p * 10)(*[f.ctypes.data for f in frames])
    op = (C.c_void_p * 10)(*[o.ctypes.data for o in outs])
    lens = (C.c_size_t * 10)()
    assert L.dfb_extract_frames_host(h, fp, 10, 64, 48, 0, 0, 95, op, cap, lens) == _lib.DFB_OK
    lengths = list(lens)
    assert L.dfb_extract_frames_host(h, fp, 0, 64, 48, 0, 0, 95, None, 0, None) == _lib.DFB_OK
    for args in [(None, 10, 64, 48, 0, 0, 95, op, cap, lens), (fp, -1, 64, 48, 0, 0, 95, op, cap, lens), (fp, 10, 64, 48, 0, 0, 0, op, cap, lens),
                 (fp, 10, 64, 48, 0, 0, 101, op, cap, lens), (fp, 10, 0, 48, 0, 0, 95, op, cap, lens), (fp, 10, 64, 48, 32, 0, 95, op, cap, lens),
                 (fp, 10, 64, 48, 0, 0, 95, None, cap, lens), (fp, 10, 64, 48, 0, 0, 95, op, cap, None)]:
        assert L.dfb_extract_frames_host(h, *args) == _lib.DFB_ERR_INVALID_ARG, args
    assert L.dfb_extract_frames_host(h, fp, 10, 64, 48, 65, 48, 95, op, cap, lens) == _lib.DFB_ERR_SIZE
    dev = torch.zeros(64 * 48 * 3, dtype=torch.uint8, device="cuda")
    for slot in (0, 9):
        bad = (C.c_void_p * 10)(*[f.ctypes.data for f in frames])
        bad[slot] = dev.data_ptr()
        assert L.dfb_extract_frames_host(h, bad, 10, 64, 48, 0, 0, 95, op, cap, lens) == _lib.DFB_ERR_INVALID_ARG
        assert L.dfb_extract_frames_host(h, fp, 10, 64, 48, 0, 0, 95, bad, cap, lens) == _lib.DFB_ERR_INVALID_ARG
        bad[slot] = None
        assert L.dfb_extract_frames_host(h, bad, 10, 64, 48, 0, 0, 95, op, cap, lens) == _lib.DFB_ERR_INVALID_ARG
    # one frame's bitstream over the capacity: a clean failure naming the length, nothing written past the capacity
    small = max(lengths) - 1
    first = next(i for i, n in enumerate(lengths) if n > small)
    guards = [np.full(cap + 64, 0xA5, np.uint8) for _ in frames]
    gp = (C.c_void_p * 10)(*[g.ctypes.data for g in guards])
    assert L.dfb_extract_frames_host(h, fp, 10, 64, 48, 0, 0, 95, gp, small, lens) == _lib.DFB_ERR_INVALID_ARG
    assert "frame %d needs %d bytes" % (first, lengths[first]) in _err(e)
    for g in guards:
        assert (g[small:] == 0xA5).all()
    # and the handle still works
    assert L.dfb_extract_frames_host(h, fp, 10, 64, 48, 0, 0, 95, op, cap, lens) == _lib.DFB_OK and list(lens) == lengths


def test_step_zero_still_rejected_by_the_flow_batch_calls():
    import denseflow_b200 as d
    e = d.create("tvl1", 0, 64, 48)
    frames = [np.zeros((48, 64), np.uint8)] * 3
    with pytest.raises(RuntimeError, match="step must be non-zero for flow extraction"):
        e.calc_batch(frames, step=0)
    with pytest.raises(RuntimeError, match="step must be non-zero for flow extraction"):
        e.process_bgr_batch([np.zeros((48, 64, 3), np.uint8)] * 3, step=0)


@pytest.mark.parametrize("w, h", [(1920, 1080), (341, 255), (17, 9), (1, 1), (2, 301)])
def test_max_bytes_bound_holds_for_noise_at_quality_100(w, h):
    import torch
    import denseflow_b200 as d
    e = d.create("farn", 0, 1920, 1080)
    bgr = torch.from_numpy(np.random.default_rng(w + h).integers(0, 256, (h, w, 3), dtype=np.uint8)).cuda()
    jpg = e.encode_jpeg_bgr_device(bgr, None, 100)
    bound = e._L.dfb_jpeg_max_bytes_bgr(w, h)
    print("noise q100 %dx%d: %d bytes, bound %d (%.2f)" % (w, h, len(jpg), bound, len(jpg) / bound))
    assert len(jpg) <= bound
