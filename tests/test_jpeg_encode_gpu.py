"""The exact JPEG encoder (denseflow_b200/csrc/jpeg_encode.cu) on the GPU: its files byte for byte against cv2.imencode(".jpg"),
the numpy restatement (tests/jpeg_encode_restate.py) and the committed fixture, through every entry point the handle
parameter "jpeg_exact" switches, plus the batch entry point dfb_encode_jpeg_gray_batch_device and the argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

import jpeg_encode_restate as E
from denseflow_b200 import _lib, synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_encode_cases.npz")
SMALL = list(range(1, 18)) + [31, 32, 33]
QUALITIES = (1, 50, 75, 95, 100)


def imencode(img, q=95):
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, int(q)])[1].tobytes()


def _same(got, want, what=""):
    assert got == want, (what, E.locate(got, want))


@pytest.fixture(scope="module")
def eng():
    import denseflow_b200 as d
    e = d.FarnebackOpticalFlow.create(0, 3840, 2160)
    e.set("jpeg_exact", 1)
    return e


def _gray(e, img, q):
    import torch
    return e.encode_jpeg_gray_device(torch.from_numpy(np.ascontiguousarray(img)).cuda(), q)


def _bgr(e, img, q, new_size=None):
    import torch
    return e.encode_jpeg_bgr_device(torch.from_numpy(np.ascontiguousarray(img)).cuda(), new_size, q)


def test_small_sizes_every_quality(eng):
    """every w, h in 1..17 and 31 / 32 / 33, gray and colour, qualities 1 / 50 / 75 / 95 / 100"""
    import torch
    rng = np.random.default_rng(5)
    for q in QUALITIES:
        for h in SMALL:
            for w in SMALL:
                g = rng.integers(0, 256, (h, w), dtype=np.uint8)
                _same(_gray(eng, g, q), imencode(g, q), ("gray", w, h, q))
                c = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                _same(_bgr(eng, c, q), imencode(c, q), ("bgr", w, h, q))
    torch.cuda.synchronize()


def test_golden_fixture(eng):
    """the committed fixture (cv2.imencode's files when it was made) and the restatement agree with the GPU"""
    z = np.load(GOLDEN)
    for k in sorted(z.files):
        if not k.startswith("img_"):
            continue
        name = k[4:]
        img, q, want = z[k], int(z["q_" + name]), z["jpg_" + name].tobytes()
        got = _gray(eng, img, q) if img.ndim == 2 else _bgr(eng, img, q)
        _same(got, want, name)
        _same(E.encode(img, q), want, ("restatement", name))


@pytest.mark.parametrize("w, h", [(340, 256), (1920, 1080), (2047, 1151), (3840, 2160)])
def test_large_sizes(eng, w, h):
    rng = np.random.default_rng(w)
    smooth = cv2.resize(rng.integers(0, 256, (h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8), (w, h))
    noisy = (smooth.astype(np.int16) + rng.integers(-20, 21, smooth.shape)).clip(0, 255).astype(np.uint8)
    for q in (95, 100):
        _same(_bgr(eng, noisy, q), imencode(noisy, q), ("bgr", w, h, q))
        g = np.ascontiguousarray(noisy[..., 1])
        _same(_gray(eng, g, q), imencode(g, q), ("gray", w, h, q))


def test_entropy_edge_cases(eng):
    """zero runs of 15 / 16 / 17 / 31 / 32 before a nonzero and before the block end, a last coefficient nonzero, DC
    differences of category 11, 0xFF bytes and a final flush byte of 0xFF: the restatement finds the images, cv2 pins them"""
    import jpeg_encode_cases as JC
    for name, img, q in JC.entropy_cases():
        want = imencode(img, q)
        _same(_gray(eng, img, q) if img.ndim == 2 else _bgr(eng, img, q), want, name)


def test_batch_equals_one_at_a_time(eng):
    """a mixed-content batch through dfb_encode_jpeg_gray_batch_device equals the same planes encoded one by one"""
    import torch
    rng = np.random.default_rng(9)
    h, w = 123, 201
    f0, f1, _ = synth.pair(h, w, seed=3)
    planes = [rng.integers(0, 256, (h, w), dtype=np.uint8), np.full((h, w), 77, np.uint8), f0, f1,
              cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (9, 9), 3)] * 3
    dev = torch.from_numpy(np.stack(planes)).cuda()
    for q in (50, 95):
        got = eng.encode_jpeg_gray_batch_device(dev, q)
        for i, p in enumerate(planes):
            _same(got[i], imencode(p, q), (i, q))
            _same(got[i], _gray(eng, p, q), (i, q, "single"))


def test_pitched_source_on_a_side_stream(eng):
    """planes whose rows and starts sit 1-3 bytes past alignment, on a non-default stream"""
    import torch
    rng = np.random.default_rng(11)
    h, w = 45, 67
    planes = rng.integers(0, 256, (4, h, w), dtype=np.uint8)
    for off in (1, 2, 3):
        pitch = w + 64 + off
        buf = torch.zeros(4 * (h + 1) * pitch + off, dtype=torch.uint8, device="cuda")
        view = buf[off:off + 4 * (h + 1) * pitch].view(4, h + 1, pitch)[:, :h, :w]
        view.copy_(torch.from_numpy(planes).cuda())
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            got = eng.encode_jpeg_gray_batch_device(view, 95)
        for i in range(4):
            _same(got[i], imencode(planes[i]), (off, i))


def test_capacity_too_small_then_a_call_works(eng):
    import torch
    rng = np.random.default_rng(13)
    img = rng.integers(0, 256, (64, 64), dtype=np.uint8)
    want = imencode(img, 100)
    dev = torch.from_numpy(np.stack([img, img])).cuda()
    for cap in (len(want) - 1, len(want) // 3, 700):
        with pytest.raises(RuntimeError, match=r"jpeg output buffer too small: plane 0 \(%d > %d\)" % (len(want), cap)):
            eng.encode_jpeg_gray_batch_device(dev, 100, capacity=cap)
    assert eng.encode_jpeg_gray_batch_device(dev, 100, capacity=len(want)) == [want, want]
    assert _gray(eng, img, 100) == want


def test_argument_checks(eng):
    import torch
    L, h = eng._L, eng._h
    dev = torch.zeros((2, 16, 16), dtype=torch.uint8, device="cuda")
    buf = np.empty(4096, np.uint8)
    outs = (C.c_void_p * 2)(buf.ctypes.data, buf.ctypes.data)
    lens = (C.c_size_t * 2)()
    call = lambda **k: L.dfb_encode_jpeg_gray_batch_device(  # noqa: E731
        h, k.get("planes", dev.data_ptr()), k.get("pitch", 16), k.get("stride", 256), k.get("n", 2), k.get("w", 16), k.get("h", 16),
        k.get("q", 95), k.get("outs", outs), k.get("cap", 4096), lens, None)
    assert call() == _lib.DFB_OK
    assert call(n=0, planes=None, outs=None) == _lib.DFB_OK
    for bad in (dict(n=-1), dict(planes=None), dict(outs=None), dict(w=0), dict(h=0), dict(pitch=15), dict(q=0), dict(q=101),
                dict(stride=100), dict(cap=0), dict(planes=buf.ctypes.data),
                dict(outs=(C.c_void_p * 2)(buf.ctypes.data, dev.data_ptr()))):
        assert call(**bad) == _lib.DFB_ERR_INVALID_ARG, bad
    assert call() == _lib.DFB_OK


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_parameter_get_set(alg):
    import denseflow_b200 as d
    e = d.create(alg, 0, 64, 64)
    assert e.get("jpeg_exact") == 0
    e.set("jpeg_exact", 1)
    assert e.get("jpeg_exact") == 1
    for bad in (2, -1, 0.5):
        with pytest.raises(RuntimeError):
            e.set("jpeg_exact", bad)
    assert e.get("jpeg_exact") == 1
    e.set("jpeg_exact", 0)
    assert e.get("jpeg_exact") == 0


def _colour(gray, seed=0):
    rng = np.random.default_rng(seed)
    return [np.stack([np.roll(g, 3, 1), g, 255 - np.roll(g, 5, 0)], -1).astype(np.uint8) ^ rng.integers(0, 4, g.shape + (3,), dtype=np.uint8)
            for g in gray]


CHAIN = [("tvl1", 1, 5, None), ("tvl1", -3, 9, (100, 72)), ("farn", 3, 9, None), ("farn", -1, 19, (101, 73)), ("tvl1", 1, 2, None),
         ("farn", 1, 1, None), ("tvl1", 3, 3, None), ("farn", 1, 19, None)]


@pytest.mark.parametrize("alg, step, n, resize", CHAIN)
def test_process_bgr_batch_exact(alg, step, n, resize):
    import denseflow_b200 as d
    gray = synth.stream(96, 128, max(n, 1), seed=7)[:n]
    bgr = _colour(gray)
    e = d.create(alg, 0, 128, 96)
    e.set("jpeg_exact", 1)
    out = e.process_bgr_batch(bgr, step=step, bound=20, new_size=resize)
    frames = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]
    if resize:
        frames = [cv2.resize(f, resize) for f in frames]
    m = max(n - abs(step), 0)
    assert len(out) == m
    if m == 0:
        return
    qx, qy = e.calc_batch(frames, step=step, bound=20)
    for i, (jx, jy) in enumerate(out):
        _same(jx, imencode(qx[i]), (i, "x"))
        _same(jy, imencode(qy[i]), (i, "y"))


def test_process_bgr_and_jpeg_batch_1080p_groups():
    """several groups in flight at 1080p (TV-L1), and the `-if` chain on imdecode'd frames"""
    import denseflow_b200 as d
    gray = synth.stream(1080, 1920, 12, seed=2)
    bgr = _colour(gray, 1)
    e = d.create("tvl1", 0, 1920, 1080)
    e.set("jpeg_exact", 1)
    out = e.process_bgr_batch(bgr, step=1, bound=20, quality=90)
    qx, qy = e.calc_batch([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr], step=1, bound=20)
    for i, (jx, jy) in enumerate(out):
        _same(jx, imencode(qx[i], 90), (i, "x"))
        _same(jy, imencode(qy[i], 90), (i, "y"))
    files = [imencode(f) for f in bgr[:6]]
    dec = [cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR) for f in files]
    out = e.process_jpeg_batch(files, step=2, bound=15, new_size=(340, 256))
    qx, qy = e.calc_batch([cv2.resize(cv2.cvtColor(f, cv2.COLOR_BGR2GRAY), (340, 256)) for f in dec], step=2, bound=15)
    for i, (jx, jy) in enumerate(out):
        _same(jx, imencode(qx[i]), (i, "x jpeg"))
        _same(jy, imencode(qy[i]), (i, "y jpeg"))


@pytest.mark.parametrize("src, dst", [((64, 48), None), ((63, 47), None), ((640, 360), (340, 256)), ((640, 360), (339, 255)),
                                      ((1920, 1080), (340, 256)), ((1920, 1080), None)])
def test_extract_frames_exact(eng, src, dst):
    sw, sh = src
    gray = synth.stream(sh, sw, 11, seed=sw)
    bgr = _colour(gray, 4)
    got = eng.extract_frames(bgr, dst, 95)
    for i, f in enumerate(bgr):
        _same(got[i], imencode(cv2.resize(f, dst) if dst else f), (i, src, dst))


def test_nvjpeg_path_unchanged_around_exact_calls():
    """on one handle, jpeg_exact = 0 gives the same bytes and flows before and after exact calls, and exact calls never
    change the flows"""
    import denseflow_b200 as d
    gray = synth.stream(96, 128, 5, seed=8)
    bgr = _colour(gray, 2)
    e = d.create("tvl1", 0, 128, 96)
    frames = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]
    before = e.process_bgr_batch(bgr, step=1, bound=20)
    fl0 = e.calc_batch(frames, step=1)
    e.set("jpeg_exact", 1)
    exact = e.process_bgr_batch(bgr, step=1, bound=20)
    fl1 = e.calc_batch(frames, step=1)
    e.set("jpeg_exact", 0)
    after = e.process_bgr_batch(bgr, step=1, bound=20)
    fl2 = e.calc_batch(frames, step=1)
    assert before == after
    assert np.array_equal(fl0, fl1) and np.array_equal(fl0, fl2)
    qx, qy = e.calc_batch(frames, step=1, bound=20)
    assert [x for x, _ in exact] == [imencode(q) for q in qx]


def _ptrs(arrs):
    return (C.c_void_p * max(len(arrs), 1))(*[a.ctypes.data for a in arrs])


def _unstuffed(f):
    """the file's length without the zeros stuffed after 0xFF data bytes (the header holds no 0xFF 0x00)"""
    return len(f) - f.count(b"\xff\x00")


def _first_over(files, cap):
    return next((i, len(f)) for i, f in enumerate(files) if len(f) > cap)


@pytest.mark.parametrize("entry", ["bgr", "jpeg"])
def test_chain_capacity_too_small_over_several_groups(entry):
    """a capacity too small for files of a group that is finished while the next group's encode is still in flight: the
    message names the exact length the first file that does not fit needs, and the next call on the handle works"""
    import denseflow_b200 as d
    gray = synth.stream(96, 128, 20, seed=12)
    gray[10] = np.random.default_rng(0).integers(0, 256, gray[10].shape, dtype=np.uint8)  # pairs 9 and 10 hold large files
    bgr = _colour(gray, 3)
    e = d.create("tvl1", 0, 128, 96)
    e.set("jpeg_exact", 1)
    if entry == "jpeg":
        src = [imencode(f) for f in bgr]
        frames = [cv2.cvtColor(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY) for f in src]
    else:
        frames = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]
    qx, qy = e.calc_batch(frames, step=1, bound=20)
    files = [imencode(p) for pair in zip(qx, qy) for p in pair]  # the order the chain checks them: x0, y0, x1, y1, ...
    m = len(qx)
    big = max(len(f) for f in files[18:22])
    small = max(len(f) for k, f in enumerate(files) if not 18 <= k < 22)
    assert small < min(_unstuffed(f) for f in files[18:22])  # the large files overflow before their stuffed zeros are counted
    assert big > small
    for cap in (small, 300):
        k, need = _first_over(files, cap)
        bx = [np.empty(cap, np.uint8) for _ in range(m)]
        by = [np.empty(cap, np.uint8) for _ in range(m)]
        lx, ly = (C.c_size_t * m)(), (C.c_size_t * m)()
        if entry == "bgr":
            rc = e._L.dfb_process_bgr_batch_host(e._h, _ptrs(bgr), len(bgr), 1, 128, 96, 0, 0, 20, 95, _ptrs(bx), _ptrs(by), cap, lx, ly)
        else:
            keep, ptrs, lens = e._jpeg_buffers(src)
            rc = e._L.dfb_process_jpeg_batch_host(e._h, ptrs, lens, len(src), 1, 0, 0, 20, 95, _ptrs(bx), _ptrs(by), cap, lx, ly)
        assert rc != _lib.DFB_OK
        msg = e._L.dfb_last_error(e._h).decode()
        assert "jpeg output buffer too small (%d > %d)" % (need, cap) in msg, (k, msg)
    out = e.process_bgr_batch(bgr, step=1, bound=20) if entry == "bgr" else e.process_jpeg_batch(src, step=1, bound=20)
    assert [f for pair in out for f in pair] == files


def test_extract_capacity_too_small_over_several_groups(eng):
    """the same for dfb_extract_frames_host: frame 10 (second group of 8, the third in flight) does not fit"""
    gray = synth.stream(64, 96, 20, seed=13)
    gray[10] = np.random.default_rng(1).integers(0, 256, gray[10].shape, dtype=np.uint8)
    bgr = _colour(gray, 5)
    files = [imencode(f) for f in bgr]
    small = max(len(f) for k, f in enumerate(files) if k != 10)
    assert small < _unstuffed(files[10])  # frame 10 overflows before its stuffed zeros are counted
    for cap, (k, need) in ((small, (10, len(files[10]))), (200, (0, len(files[0])))):
        outs = [np.empty(cap, np.uint8) for _ in bgr]
        lens = (C.c_size_t * len(bgr))()
        rc = eng._L.dfb_extract_frames_host(eng._h, _ptrs(bgr), len(bgr), 96, 64, 0, 0, 95, _ptrs(outs), cap, lens)
        assert rc != _lib.DFB_OK
        msg = eng._L.dfb_last_error(eng._h).decode()
        assert "frame %d needs %d bytes, capacity is %d" % (k, need, cap) in msg, msg
    assert eng.extract_frames(bgr, None, 95) == files
