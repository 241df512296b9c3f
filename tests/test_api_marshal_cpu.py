"""No-GPU checks of the Python bindings' marshalling: api.DenseOpticalFlow's host batch methods and listrun's entry points run
against a fake library that records every dfb_* call (its scalars, the length and order of each pointer array and which
buffer each pointer names) and writes deterministic outputs through the pointers and length arrays it is given.  Each test
pins the recorded calls, the returned shapes, dtypes and bytes, and the text of every refusal the Python side makes."""
import ctypes as C

import numpy as np
import pytest

from denseflow_b200 import _lib, api, listrun

H, W = 6, 8          # frame size of the flow tests
MW, MH = 40, 30      # the handle's maximum frame
JW, JH = 10, 7       # the size dfb_jpeg_info reports
HANDLE = 0x5000    # the fake engine handle
NOT_RECORDED = {"dfb_last_error", "dfb_destroy", "dfb_list_close"}


def m_of(n, step):
    return max(n - abs(step), 0)


# what the fake writes: pair i's field, u8 plane c, float plane c, and file c of item i of the call named `fn`
def field(i, h, w):
    return (np.arange(h * w * 2, dtype=np.float32) + 1000 * i).reshape(h, w, 2)


def u8(i, c, h, w):
    return ((np.arange(h * w) + 7 * i + 100 * c) % 251).astype(np.uint8).reshape(h, w)


def plane(i, c, h, w):
    return (np.arange(h * w, dtype=np.float32) * (c + 1) + 1000 * i).reshape(h, w)


def file(fn, c, i):
    return bytes((len(fn) + 31 * c + 7 * i + j) % 256 for j in range(5 + 3 * i + c))


def jpeg_cap(w, h):
    return w * h + 64


def png_cap(w, h):
    return 2 * w * h + 50


def bgr_cap(w, h):
    return 3 * w * h + 60


class FakeLib:
    """Stands in for the CUDA library behind _lib.load: every symbol of _lib.SIGNATURES, called with its arity."""

    def __init__(self):
        self.calls = []
        self.params = {}
        self.error = b""
        self.fail = {}  # name -> (rc, message): the next call of that name fails so

    def __getattr__(self, name):
        if name not in _lib.SIGNATURES:
            raise AttributeError(name)
        impl = getattr(self, "on_" + name, None)

        def call(*args):
            assert len(args) == len(_lib.SIGNATURES[name][1]), (name, len(args))
            if name in NOT_RECORDED:
                return impl(*args) if impl else None
            self.calls.append((name, args))
            if name in self.fail:
                rc, self.error = self.fail.pop(name)
                return rc
            return impl(*args) if impl else 0
        return call

    def refuse(self, msg):
        self.error = msg.encode()
        return _lib.DFB_ERR_INVALID_ARG

    # -- the handle --
    def on_dfb_create(self, alg, dev, mw, mh, out):
        out._obj.value = HANDLE
        return 0

    def on_dfb_last_error(self, h):
        return self.error

    def on_dfb_set_param(self, h, name, value):
        self.params[name] = value
        return 0

    def on_dfb_get_param(self, h, name, out):
        out._obj.value = self.params.get(name, 0.0)
        return 0

    def on_dfb_jpeg_max_bytes(self, w, h):
        return jpeg_cap(w, h)

    def on_dfb_png_max_bytes(self, w, h):
        return png_cap(w, h)

    def on_dfb_jpeg_max_bytes_bgr(self, w, h):
        return bgr_cap(w, h)

    def on_dfb_jpeg_info(self, ptr, n, w, h):
        w._obj.value, h._obj.value = JW, JH
        return 0

    # -- outputs --
    @staticmethod
    def put(addr, a):
        C.memmove(addr, a.ctypes.data, a.nbytes)

    def fields(self, op, m, h, w):
        if op is None:
            return self.refuse("flows is null")
        for i in range(m):
            self.put(op[i], field(i, h, w))
        return 0

    def u8s(self, xp, yp, m, h, w):
        for c, p in enumerate((xp, yp)):
            for i in range(m):
                self.put(p[i], u8(i, c, h, w))
        return 0

    def planes(self, xp, yp, m, h, w):
        if xp is None or yp is None:
            return self.refuse("fx/fy is null")
        for c, p in enumerate((xp, yp)):
            for i in range(m):
                self.put(p[i], plane(i, c, h, w))
        return 0

    def files(self, fn, ptrs, cap, lens, m):
        for c, (p, ln) in enumerate(zip(ptrs, lens)):
            for i in range(m):
                b = file(fn, c, i)
                assert len(b) <= cap
                C.memmove(p[i], b, len(b))
                ln[i] = len(b)
        return 0

    @staticmethod
    def out_size(dw, dh, w, h):
        return (dh, dw) if dw else (h, w)

    def on_dfb_calc_host(self, hd, a, b, w, h, flow):
        if flow is None:
            return self.refuse("null buffer")
        self.put(flow, field(0, h, w))
        return 0

    def on_dfb_calc_batch_host(self, hd, fp, n, step, w, h, op):
        return self.fields(op, m_of(n, step), h, w)

    def on_dfb_calc_batch_host_u8(self, hd, fp, n, step, w, h, bound, xp, yp):
        return self.u8s(xp, yp, m_of(n, step), h, w)

    def on_dfb_calc_batch_host_planes(self, hd, fp, n, step, w, h, xp, yp):
        return self.planes(xp, yp, m_of(n, step), h, w)

    def on_dfb_calc_batch_host_png(self, hd, fp, n, step, w, h, op, cap, lens):
        return self.files("dfb_calc_batch_host_png", [op], cap, [lens], m_of(n, step))

    def on_dfb_process_bgr_batch_host(self, hd, fp, n, step, sw, sh, dw, dh, bound, q, xp, yp, cap, lx, ly):
        return self.files("dfb_process_bgr_batch_host", [xp, yp], cap, [lx, ly], m_of(n, step))

    def on_dfb_process_bgr_batch_host_png(self, hd, fp, n, step, sw, sh, dw, dh, op, cap, lens):
        return self.files("dfb_process_bgr_batch_host_png", [op], cap, [lens], m_of(n, step))

    def on_dfb_process_bgr_batch_host_planes(self, hd, fp, n, step, sw, sh, dw, dh, xp, yp):
        return self.planes(xp, yp, m_of(n, step), *self.out_size(dw, dh, sw, sh))

    def on_dfb_process_jpeg_batch_host(self, hd, ptrs, lens, n, step, dw, dh, bound, q, xp, yp, cap, lx, ly):
        return self.files("dfb_process_jpeg_batch_host", [xp, yp], cap, [lx, ly], m_of(n, step))

    def on_dfb_process_jpeg_batch_host_png(self, hd, ptrs, lens, n, step, dw, dh, op, cap, olens):
        return self.files("dfb_process_jpeg_batch_host_png", [op], cap, [olens], m_of(n, step))

    def on_dfb_process_jpeg_batch_host_planes(self, hd, ptrs, lens, n, step, dw, dh, xp, yp):
        return self.planes(xp, yp, m_of(n, step), *self.out_size(dw, dh, JW, JH))

    def on_dfb_extract_frames_host(self, hd, fp, n, sw, sh, dw, dh, q, op, cap, lens):
        return self.files("dfb_extract_frames_host", [op], cap, [lens], n)

    def on_dfb_extract_frames_jpeg_host(self, hd, ptrs, lens, n, dw, dh, q, op, cap, olens):
        return self.files("dfb_extract_frames_jpeg_host", [op], cap, [olens], n)

    # -- the list runner --
    def on_dfb_list_open(self, alg, devs, ndev, mw, mh, out, err, err_len):
        out._obj.value = 0x6000
        return 0

    @staticmethod
    def stats(st):
        s = st._obj
        s.clips, s.flows, s.frames, s.seconds, s.workers = 3, 5, 8, 1.5, 2
        for k in range(2):
            s.clips_per_worker[k], s.flows_per_worker[k] = 1 + k, 2 + k
            s.busy_seconds_per_worker[k], s.finish_seconds_per_worker[k] = 0.25 + k, 0.5 + k
        s.kernel_launches, s.h2d_bytes, s.d2h_bytes = 7, 11, 13
        return 0

    def chunks(self, cb, clips, n_clips):
        """one chunk per clip: flows 0 .. n - 2 of clip k as two u8 planes or a float2 field each"""
        if cb is None:
            return
        fn = _lib.CHUNK_DONE_FN(cb.value if isinstance(cb, C.c_void_p) else cb)
        for k in range(n_clips):
            h, w, m = clips[k].height, clips[k].width, clips[k].n_frames - 1
            bufs = [u8(i, c, h, w) for c in range(2) for i in range(m)] + [field(i, h, w) for i in range(m)]
            ptr = [(C.c_void_p * max(m, 1))(*[b.ctypes.data for b in bufs[j * m:(j + 1) * m]]) for j in range(3)]
            quant = self.params.get("bound", 1)
            fn(None, k, 0, 0, m, 1, ptr[0] if quant else None, ptr[1] if quant else None, None if quant else ptr[2])

    def on_dfb_list_run(self, r, clips, n, step, bound, chunk, queue, cb, user, st, err, err_len):
        self.params["bound"] = bound
        self.chunks(cb, clips, n)
        return self.stats(st)

    def on_dfb_run_list(self, alg, devs, ndev, clips, n, step, bound, chunk, queue, cb, user, st, err, err_len):
        self.params["bound"] = bound
        self.chunks(cb, clips, n)
        return self.stats(st)

    def files_done(self, cb, video, n, per):
        """one chunk of n flows (per files each) of `video`"""
        if cb is None:
            return
        bufs = [file("list", j % per, j // per) for j in range(per * n)]
        ptrs = (C.c_void_p * max(len(bufs), 1))(*[C.cast(C.c_char_p(b), C.c_void_p).value for b in bufs])
        lens = (C.c_size_t * max(len(bufs), 1))(*[len(b) for b in bufs])
        _lib.FILES_DONE_FN(cb.value)(None, video, 1, 2, n, 1, ptrs, lens)

    def on_dfb_list_run_videos(self, r, videos, n, step, bound, save, q, exact, nw, nh, ns, chunk, queue, cb, user, st, err,
                               err_len):
        self.videos = [(videos[k].kind, videos[k].n_frames, videos[k].width, videos[k].height) for k in range(n)]
        for k in range(n):
            self.files_done(cb, k, videos[k].n_frames - 1, 2 if step != 0 and save != _lib.SAVE_PNG else 1)
        return self.stats(st)

    def run_source(self, n, src, step, save, cb, st, err):
        fn = _lib.FRAMES_FN(src.value)
        self.videos = []
        for k in range(n):
            v = _lib.Video()
            msg = C.create_string_buffer(64)
            if fn(None, k, 0, 4, C.pointer(v), C.cast(msg, C.c_void_p), 64):
                err.value = b"video %d: " % k + msg.value
                return _lib.DFB_ERR_INVALID_ARG
            self.videos.append((v.kind, v.n_frames, v.width, v.height))
            self.files_done(cb, k, v.n_frames - 1, 2 if step != 0 and save != _lib.SAVE_PNG else 1)
        return self.stats(st)

    def on_dfb_list_run_stream(self, r, n, src, step, bound, save, q, exact, nw, nh, ns, chunk, queue, cb, user, st, err, err_len):
        return self.run_source(n, src, step, save, cb, st, err)

    def on_dfb_list_run_windows(self, r, n, src, step, bound, save, q, exact, nw, nh, ns, chunk, queue, cb, user, st, err,
                                err_len):
        return self.run_source(n, src, step, save, cb, st, err)


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda variant="default": f)
    return f


@pytest.fixture
def e(fake):
    eng = api.OpticalFlowDual_TVL1.create(0, MW, MH)
    assert fake.calls == [("dfb_create", (b"tvl1", 0, MW, MH, fake.calls[0][1][4]))]
    fake.calls.clear()
    return eng


def addr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else np.frombuffer(a, np.uint8).ctypes.data if isinstance(a, bytes) else a.ctypes.data


def labels(**named):
    """address -> "name[i]" for every buffer of the given lists"""
    return {addr(b): "%s[%d]" % (k, i) for k, bufs in named.items() for i, b in enumerate(bufs)}


def desc(x, lab):
    if isinstance(x, C.Array):
        if x._type_ is C.c_void_p:
            return [None if p is None else lab.get(p, "new") for p in x]
        if x._type_ is C.c_size_t:
            return ("size_t", len(x))
        if x._type_ is C.c_char:
            return ("err", len(x))
        return (x._type_.__name__, len(x))
    if type(x).__name__ == "CArgObject":
        return ("byref", type(x._obj).__name__)
    if isinstance(x, C.c_void_p):
        return ("stream", x.value)
    if isinstance(x, int) and x in lab:
        return lab[x]
    return x


def is_handle(x):
    return isinstance(x, C.c_void_p) and x.value == HANDLE


def log(fake, **named):
    lab = labels(**named)
    out = [(name,) + tuple(desc(a, lab) for a in (args[1:] if is_handle(args[0]) else args)) for name, args in fake.calls]
    fake.calls.clear()
    return out


def gray(n, h=H, w=W, seed=0):
    r = np.random.default_rng(seed)
    return [r.integers(0, 256, (h, w), dtype=np.uint8) for _ in range(n)]


def bgr(n, h=H, w=W, seed=1):
    r = np.random.default_rng(seed)
    return [r.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]


def jpegs(n):
    return [b"\xff\xd8jpeg%d" % i for i in range(n)]


def rows(a):
    return [a[i] for i in range(a.shape[0])]


NEW = "new"


# -- calc / calc_batch / calc_batch_u8_into --

def test_calc_host(e, fake):
    a, b = gray(2)
    flow = e.calc(a, b)
    assert flow.dtype == np.float32 and flow.shape == (H, W, 2) and np.array_equal(flow, field(0, H, W))
    assert log(fake, f=[a, b], o=[flow]) == [("dfb_get_param", b"use_initial_flow", ("byref", "c_double")),
                                             ("dfb_calc_host", "f[0]", "f[1]", W, H, "o[0]")]
    given = np.zeros((H, W, 2), np.float32)
    assert e.calc(a, b, flow=given) is given and np.array_equal(given, field(0, H, W))
    assert log(fake, f=[a, b], o=[given]) == [("dfb_calc_host", "f[0]", "f[1]", W, H, "o[0]")]
    with pytest.raises(RuntimeError, match=r"^calc: frames must be two CV_8UC1 images of the same size$"):
        e.calc(a, b[:, :4])
    e.set("use_initial_flow", 1)
    with pytest.raises(RuntimeError, match="^null buffer$"):
        e.calc(a, b)
    assert log(fake, f=[a, b])[-1] == ("dfb_calc_host", "f[0]", "f[1]", W, H, None)


@pytest.mark.parametrize("n,step", [(5, 1), (5, -2), (2, 3), (1, 1)])
def test_calc_batch_field(e, fake, n, step):
    fr = gray(n)
    m = m_of(n, step)
    flows = e.calc_batch(fr, step)
    assert flows.dtype == np.float32 and flows.shape == (m, H, W, 2)
    assert all(np.array_equal(flows[i], field(i, H, W)) for i in range(m))
    want = [("dfb_get_param", b"use_initial_flow", ("byref", "c_double")),
            ("dfb_calc_batch_host", ["f[%d]" % i for i in range(n)], n, step, W, H, ["o[%d]" % i for i in range(m)] or [None])]
    assert log(fake, f=fr, o=rows(flows)) == want
    # a caller's array (more rows than pairs is fine), and one [N,H,W] array as the frames
    given = np.zeros((m + 1, H, W, 2), np.float32)
    stack = np.stack(fr)
    assert e.calc_batch(stack, step, flows=given) is given
    assert all(np.array_equal(given[i], field(i, H, W)) for i in range(m)) and not given[m].any()
    assert log(fake, f=rows(stack), o=rows(given)) == [want[1][:6] + (["o[%d]" % i for i in range(m)] or [None],)]


def test_calc_batch_refusals(e, fake):
    fr = gray(3)
    with pytest.raises(RuntimeError, match=r"^frame 2: expected a uint8 \[H,W\] image of the same size as frame 0$"):
        e.calc_batch(fr[:2] + [fr[2][:, :5]])
    with pytest.raises(RuntimeError, match=r"^frame 1: expected a uint8 \[H,W\] image of the same size as frame 0$"):
        e.calc_batch([fr[0], fr[1].astype(np.int16)])
    with pytest.raises(RuntimeError, match=r"^frame 0: expected"):
        e.calc_batch([np.zeros((2, 3, 1), np.uint8)])
    for bad in [np.zeros((1, H, W, 2), np.float32), np.zeros((2, H, W, 2), np.float64), np.zeros((2, H, W + 1, 2), np.float32),
                np.zeros((2, H, W, 4), np.float32)[..., :2], [np.zeros((H, W, 2), np.float32)] * 2]:
        with pytest.raises(RuntimeError, match=r"^flows: expected a C-contiguous float32 array of shape \(2, 6, 8, 2\)$"):
            e.calc_batch(fr, 1, flows=bad)
    assert [c[0] for c in fake.calls if c[0] != "dfb_get_param"] == []
    fake.calls.clear()
    fake.fail = {"dfb_calc_batch_host": (_lib.DFB_ERR_CUDA, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb error -3$"):
        e.calc_batch(fr, 1, flows=np.zeros((2, H, W, 2), np.float32))
    fake.fail = {"dfb_calc_batch_host": (_lib.DFB_ERR_SIZE, b"frame size 8x6 exceeds the handle")}
    with pytest.raises(RuntimeError, match=r"^frame size 8x6 exceeds the handle$"):
        e.calc_batch(fr, 1, flows=np.zeros((2, H, W, 2), np.float32))


def test_calc_batch_empty(e, fake):
    for kw in ({}, {"bound": 20}, {"flows": np.zeros((1, 1, 1, 2), np.float32)}):
        out = e.calc_batch([], 1, **kw)
        assert isinstance(out, np.ndarray) and out.shape == (0, 0, 0, 2) and out.dtype == np.float32
    assert e.calc_batch_planes([], 1).shape == (0, 2, 0, 0)
    assert e.calc_batch_planes(np.zeros((0, H, W), np.uint8), 1).dtype == np.float32
    assert e.calc_batch_png([], 1) == []
    with pytest.raises(IndexError):
        e.calc_batch_u8_into([], 1, 20, np.zeros((0, H, W), np.uint8), np.zeros((0, H, W), np.uint8))
    assert fake.calls == []


@pytest.mark.parametrize("n,step,bound", [(4, 1, 20), (4, -3, 7), (2, 2, 20)])
def test_calc_batch_u8(e, fake, n, step, bound):
    fr = gray(n)
    m = m_of(n, step)
    qx, qy = e.calc_batch(fr, step, bound=bound)
    for c, q in enumerate((qx, qy)):
        assert q.dtype == np.uint8 and q.shape == (m, H, W)
        assert all(np.array_equal(q[i], u8(i, c, H, W)) for i in range(m))
    ptrs = lambda k: ["%s[%d]" % (k, i) for i in range(m)] or [None]  # noqa: E731
    want = [("dfb_calc_batch_host_u8", ["f[%d]" % i for i in range(n)], n, step, W, H, bound, ptrs("x"), ptrs("y"))]
    assert log(fake, f=fr, x=rows(qx), y=rows(qy)) == want
    px, py = np.zeros((m + 2, H, W), np.uint8), np.zeros((m, H, W), np.uint8)
    got = e.calc_batch_u8_into(fr, step, bound, px, py)
    assert got[0] is px and got[1] is py
    assert all(np.array_equal(px[i], u8(i, 0, H, W)) and np.array_equal(py[i], u8(i, 1, H, W)) for i in range(m))
    assert log(fake, f=fr, x=rows(px), y=rows(py)) == want


def test_calc_batch_u8_into_refusals(e, fake):
    fr = gray(3)
    ok = np.zeros((2, H, W), np.uint8)
    for bad in [np.zeros((1, H, W), np.uint8), np.zeros((2, H, W), np.int8), np.zeros((2, W, H), np.uint8), list(ok)]:
        with pytest.raises(RuntimeError, match=r"^qx: expected a C-contiguous uint8 array of shape \(2, 6, 8\)$"):
            e.calc_batch_u8_into(fr, 1, 20, bad, ok)
        with pytest.raises(RuntimeError, match=r"^qy: expected a C-contiguous uint8 array of shape \(2, 6, 8\)$"):
            e.calc_batch_u8_into(fr, 1, 20, ok, bad)
    with pytest.raises(RuntimeError, match=r"^frame 1: expected"):
        e.calc_batch_u8_into([fr[0], fr[1][:3]], 1, 20, ok, ok)
    assert fake.calls == []


# -- use_initial_flow: the probe for a missing flow buffer --

def test_warm_start_probe(e, fake):
    fr = gray(3)
    e.set("use_initial_flow", 1)
    assert log(fake) == [("dfb_set_param", b"use_initial_flow", 1.0)]
    get = ("dfb_get_param", b"use_initial_flow", ("byref", "c_double"))
    with pytest.raises(RuntimeError, match="^flows is null$"):
        e.calc_batch(fr, 1)
    assert log(fake, f=fr) == [get, ("dfb_calc_batch_host", ["f[0]", "f[1]", "f[2]"], 3, 1, W, H, None)]
    with pytest.raises(RuntimeError, match="^fx/fy is null$"):
        e.calc_batch_planes(fr, 1)
    assert log(fake, f=fr) == [get, ("dfb_calc_batch_host_planes", ["f[0]", "f[1]", "f[2]"], 3, 1, W, H, None, None)]
    # no pairs: nothing is read, so no probe; the call runs with fresh outputs
    flows = e.calc_batch(fr, 3)
    assert flows.shape == (0, H, W, 2)
    assert log(fake, f=fr) == [get, ("dfb_calc_batch_host", ["f[0]", "f[1]", "f[2]"], 3, 3, W, H, [None])]
    planes = e.calc_batch_planes(fr, -4)
    assert planes.shape == (0, 2, H, W)
    assert log(fake, f=fr) == [get, ("dfb_calc_batch_host_planes", ["f[0]", "f[1]", "f[2]"], 3, -4, W, H, [None], [None])]
    # with the buffers given, no probe
    given = np.ones((2, H, W, 2), np.float32)
    assert e.calc_batch(fr, 1, flows=given) is given
    assert log(fake, f=fr, o=rows(given)) == [("dfb_calc_batch_host", ["f[0]", "f[1]", "f[2]"], 3, 1, W, H, ["o[0]", "o[1]"])]
    e.set("use_initial_flow", 0)
    fake.calls.clear()
    flows = e.calc_batch(fr, 1)
    assert [c[0] for c in log(fake)] == ["dfb_get_param", "dfb_calc_batch_host"]


# -- float planes --

@pytest.mark.parametrize("n,step", [(4, 1), (4, -2), (2, 5)])
def test_calc_batch_planes(e, fake, n, step):
    fr = gray(n)
    m = m_of(n, step)
    out = e.calc_batch_planes(fr, step)
    assert out.dtype == np.float32 and out.shape == (m, 2, H, W)
    assert all(np.array_equal(out[i, c], plane(i, c, H, W)) for i in range(m) for c in range(2))
    xs = lambda c: ["o[%d]" % (2 * i + c) for i in range(m)] or [None]  # noqa: E731
    want = ("dfb_calc_batch_host_planes", ["f[%d]" % i for i in range(n)], n, step, W, H)
    flat = lambda a: [a[i, c] for i in range(a.shape[0]) for c in range(2)]  # noqa: E731
    assert log(fake, f=fr, o=flat(out)) == [("dfb_get_param", b"use_initial_flow", ("byref", "c_double")),
                                            want + (xs(0), xs(1))]
    given = np.zeros((m + 1, 2, H, W), np.float32)
    assert e.calc_batch_planes(fr, step, out=given) is given
    assert log(fake, f=fr, o=flat(given)) == [want + (xs(0), xs(1))]
    with pytest.raises(RuntimeError, match=r"^out: expected a C-contiguous float32 array of shape \(%d, 2, 6, 8\)$" % m):
        e.calc_batch_planes(fr, step, out=np.zeros((m + 1, H, W, 2), np.float32))


@pytest.mark.parametrize("new_size", [None, (5, 4), [12, 9]])
def test_process_bgr_batch_planes(e, fake, new_size):
    fr = bgr(4)
    out = e.process_bgr_batch_planes(fr, 1, new_size)
    oh, ow = (new_size[1], new_size[0]) if new_size else (H, W)
    assert out.dtype == np.float32 and out.shape == (3, 2, oh, ow)
    assert all(np.array_equal(out[i, c], plane(i, c, oh, ow)) for i in range(3) for c in range(2))
    dw, dh = new_size or (0, 0)
    assert log(fake, f=fr, o=[out[i, c] for i in range(3) for c in range(2)]) == [
        ("dfb_process_bgr_batch_host_planes", ["f[0]", "f[1]", "f[2]", "f[3]"], 4, 1, W, H, dw, dh, ["o[0]", "o[2]", "o[4]"],
         ["o[1]", "o[3]", "o[5]"])]
    assert e.process_bgr_batch_planes(fr[:1], 1).shape == (0, 2, H, W)
    assert log(fake, f=fr[:1]) == [("dfb_process_bgr_batch_host_planes", ["f[0]"], 1, 1, W, H, 0, 0, [None], [None])]
    assert e.process_bgr_batch_planes([], 1, new_size).shape == (0, 2, 0, 0)
    with pytest.raises(RuntimeError, match=r"^process_bgr_batch_planes: frames must be uint8 \[H,W,3\] images of one size$"):
        e.process_bgr_batch_planes([fr[0], fr[1].astype(np.float32)])
    assert fake.calls == []


@pytest.mark.parametrize("new_size,step", [(None, 1), ((5, 4), -2), (None, 9)])
def test_process_jpeg_batch_planes(e, fake, new_size, step):
    files = jpegs(4)
    m = m_of(4, step)
    out = e.process_jpeg_batch_planes(files, step, new_size)
    oh, ow = (new_size[1], new_size[0]) if new_size else (JH, JW)
    assert out.dtype == np.float32
    if m == 0:
        assert out.shape == (0, 2, 0, 0) and fake.calls == []
        return
    assert out.shape == (m, 2, oh, ow)
    assert all(np.array_equal(out[i, c], plane(i, c, oh, ow)) for i in range(m) for c in range(2))
    dw, dh = new_size or (0, 0)
    info = [] if new_size else [("dfb_jpeg_info", "j[0]", len(files[0]), ("byref", "c_int"), ("byref", "c_int"))]
    assert log(fake, j=files, o=[out[i, c] for i in range(m) for c in range(2)]) == info + [
        ("dfb_process_jpeg_batch_host_planes", ["j[0]", "j[1]", "j[2]", "j[3]"], ("size_t", 4), 4, step, dw, dh,
         ["o[%d]" % (2 * i) for i in range(m)], ["o[%d]" % (2 * i + 1) for i in range(m)])]


def test_process_jpeg_batch_planes_info_refusal(e, fake):
    fake.fail = {"dfb_jpeg_info": (_lib.DFB_ERR_INVALID_ARG, b"not a JPEG file")}
    with pytest.raises(RuntimeError, match="^not a JPEG file$"):
        e.process_jpeg_batch_planes(jpegs(3))
    assert [c[0] for c in fake.calls] == ["dfb_jpeg_info"]


# -- files: JPEG pairs, PNG per pair, JPEG per frame --

def pairs_of(fn, m):
    return [(file(fn, 0, i), file(fn, 1, i)) for i in range(m)]


def singles_of(fn, m):
    return [file(fn, 0, i) for i in range(m)]


@pytest.mark.parametrize("new_size,step", [(None, 1), ((5, 4), 2), (None, -7)])
def test_process_bgr_batch(e, fake, new_size, step):
    fr = bgr(5)
    m = m_of(5, step)
    out = e.process_bgr_batch(fr, step, 15, new_size, 90)
    assert out == pairs_of("dfb_process_bgr_batch_host", m) and all(isinstance(f, bytes) for p in out for f in p)
    ow, oh = new_size or (W, H)
    dw, dh = new_size or (0, 0)
    new = [NEW] * m or [None]
    assert log(fake, f=fr) == [("dfb_jpeg_max_bytes", ow, oh),
                               ("dfb_process_bgr_batch_host", ["f[%d]" % i for i in range(5)], 5, step, W, H, dw, dh, 15, 90, new,
                                new, jpeg_cap(ow, oh), ("size_t", max(m, 1)), ("size_t", max(m, 1)))]


def test_process_bgr_batch_frames(e, fake):
    # process_bgr_batch converts any dtype to uint8 and takes non-contiguous frames; the other BGR entries refuse a non-uint8 frame
    fr = [f.astype(np.float32) for f in bgr(3)]
    fr[1] = np.ascontiguousarray(bgr(1)[0][:, ::-1]).astype(np.int64)[:, ::-1]
    assert e.process_bgr_batch(fr) == pairs_of("dfb_process_bgr_batch_host", 2)
    assert [c[0] for c in log(fake)] == ["dfb_jpeg_max_bytes", "dfb_process_bgr_batch_host"]
    with pytest.raises(RuntimeError, match=r"^process_bgr_batch_png: frames must be uint8 \[H,W,3\] images of one size$"):
        e.process_bgr_batch_png(fr)
    with pytest.raises(RuntimeError, match=r"^extract_frames: frames must be uint8 \[H,W,3\] images of one size$"):
        e.extract_frames(fr)
    good = bgr(2)
    for bad in [good + [good[0][:, :, :2]], good + [good[0][:5]], good + [good[0][:, :, 0]]]:
        with pytest.raises(RuntimeError, match=r"^process_bgr_batch: frames must be uint8 \[H,W,3\] images of one size$"):
            e.process_bgr_batch(bad)
    with pytest.raises(IndexError):
        e.process_bgr_batch([])
    assert fake.calls == []


@pytest.mark.parametrize("new_size,step", [(None, 1), ((5, 4), -1), (None, 4)])
def test_process_jpeg_batch(e, fake, new_size, step):
    files = jpegs(4)
    m = m_of(4, step)
    out = e.process_jpeg_batch(files, step, 25, new_size, 80)
    assert out == pairs_of("dfb_process_jpeg_batch_host", m)
    ow, oh = new_size or (MW, MH)
    dw, dh = new_size or (0, 0)
    new = [NEW] * m or [None]
    assert log(fake, j=files) == [("dfb_jpeg_max_bytes", ow, oh),
                                  ("dfb_process_jpeg_batch_host", ["j[0]", "j[1]", "j[2]", "j[3]"], ("size_t", 4), 4, step, dw, dh,
                                   25, 80, new, new, jpeg_cap(ow, oh), ("size_t", max(m, 1)), ("size_t", max(m, 1)))]


def test_process_jpeg_batch_empty(e, fake):
    assert e.process_jpeg_batch([]) == []
    assert log(fake) == [("dfb_jpeg_max_bytes", MW, MH),
                         ("dfb_process_jpeg_batch_host", [None], ("size_t", 1), 0, 1, 0, 0, 20, 95, [None], [None],
                          jpeg_cap(MW, MH), ("size_t", 1), ("size_t", 1))]
    assert e.process_jpeg_batch_png([]) == []
    assert [c[0] for c in log(fake)] == ["dfb_png_max_bytes", "dfb_process_jpeg_batch_host_png"]
    assert e.extract_frames_jpeg([]) == []
    assert e.process_jpeg_batch_planes([]).shape == (0, 2, 0, 0)
    assert fake.calls == []


def test_jpeg_buffer_kinds(e, fake):
    import torch
    raw = jpegs(4)
    tail = bytearray(raw[3])
    src = [raw[0], bytearray(raw[1]), np.frombuffer(raw[2], np.uint8).reshape(1, -1), torch.frombuffer(tail, dtype=torch.uint8)]
    out = e.extract_frames_jpeg(src)
    assert out == singles_of("dfb_extract_frames_jpeg_host", 4)
    (_, (_, ptrs, lens, n, *_)), = [c for c in fake.calls if c[0] == "dfb_extract_frames_jpeg_host"]
    assert ptrs[0] == addr(raw[0]) and ptrs[3] == src[3].data_ptr() and list(lens) == [len(r) for r in raw] and n == 4
    fake.calls.clear()
    with pytest.raises(RuntimeError, match="^JPEG buffers must be contiguous uint8 host memory$"):
        e.process_jpeg_batch([raw[0], torch.zeros(8, dtype=torch.int32)])
    with pytest.raises(RuntimeError, match="^JPEG buffers must be contiguous uint8 host memory$"):
        e.process_jpeg_batch_png([torch.zeros(8, dtype=torch.uint8)[::2]])
    assert fake.calls == []


@pytest.mark.parametrize("new_size,step", [(None, 1), ((5, 4), -2), (None, 3)])
def test_process_bgr_batch_png(e, fake, new_size, step):
    fr = bgr(3)
    m = m_of(3, step)
    out = e.process_bgr_batch_png(fr, step, new_size)
    assert out == singles_of("dfb_process_bgr_batch_host_png", m)
    ow, oh = new_size or (W, H)
    dw, dh = new_size or (0, 0)
    assert log(fake, f=fr) == [("dfb_png_max_bytes", ow, oh),
                               ("dfb_process_bgr_batch_host_png", ["f[0]", "f[1]", "f[2]"], 3, step, W, H, dw, dh,
                                [NEW] * m or [None], png_cap(ow, oh), ("size_t", max(m, 1)))]
    assert e.process_bgr_batch_png([], step, new_size) == [] and fake.calls == []


@pytest.mark.parametrize("new_size,step", [(None, 1), ((5, 4), 2), (None, -5)])
def test_process_jpeg_batch_png(e, fake, new_size, step):
    files = jpegs(5)
    m = m_of(5, step)
    out = e.process_jpeg_batch_png(files, step, new_size)
    assert out == singles_of("dfb_process_jpeg_batch_host_png", m)
    ow, oh = new_size or (MW, MH)
    dw, dh = new_size or (0, 0)
    assert log(fake, j=files) == [("dfb_png_max_bytes", ow, oh),
                                  ("dfb_process_jpeg_batch_host_png", ["j[%d]" % i for i in range(5)], ("size_t", 5), 5, step, dw, dh,
                                   [NEW] * m or [None], png_cap(ow, oh), ("size_t", max(m, 1)))]


@pytest.mark.parametrize("new_size", [None, (5, 4)])
def test_extract_frames(e, fake, new_size):
    fr = bgr(3)
    stack = np.stack(fr)
    for src in (fr, stack):
        out = e.extract_frames(src, new_size, 70)
        assert out == singles_of("dfb_extract_frames_host", 3)
        ow, oh = new_size or (W, H)
        dw, dh = new_size or (0, 0)
        assert log(fake, f=list(src)) == [("dfb_jpeg_max_bytes_bgr", ow, oh),
                                          ("dfb_extract_frames_host", ["f[0]", "f[1]", "f[2]"], 3, W, H, dw, dh, 70, [NEW] * 3,
                                           bgr_cap(ow, oh), ("size_t", 3))]
    assert e.extract_frames([], new_size) == [] and fake.calls == []


@pytest.mark.parametrize("new_size", [None, (5, 4)])
def test_extract_frames_jpeg(e, fake, new_size):
    files = jpegs(3)
    out = e.extract_frames_jpeg(files, new_size, 60)
    assert out == singles_of("dfb_extract_frames_jpeg_host", 3)
    ow, oh = new_size or (MW, MH)
    dw, dh = new_size or (0, 0)
    assert log(fake, j=files) == [("dfb_jpeg_max_bytes_bgr", ow, oh),
                                  ("dfb_extract_frames_jpeg_host", ["j[0]", "j[1]", "j[2]"], ("size_t", 3), 3, dw, dh, 60, [NEW] * 3,
                                   bgr_cap(ow, oh), ("size_t", 3))]


@pytest.mark.parametrize("n,step", [(4, 1), (4, -3), (2, 2)])
def test_calc_batch_png(e, fake, n, step):
    fr = gray(n)
    m = m_of(n, step)
    out = e.calc_batch_png(fr, step)
    assert out == singles_of("dfb_calc_batch_host_png", m)
    want = [("dfb_png_max_bytes", W, H),
            ("dfb_calc_batch_host_png", ["f[%d]" % i for i in range(n)], n, step, W, H, [NEW] * m or [None], png_cap(W, H),
             ("size_t", max(m, 1)))]
    assert log(fake, f=fr) == want
    # caller buffers, more of them than pairs, and a 2-D array of them
    for bufs in ([np.zeros(png_cap(W, H) + 3, np.uint8) for _ in range(m + 1)], np.zeros((m + 1, png_cap(W, H)), np.uint8)):
        assert e.calc_batch_png(fr, step, out=bufs) == singles_of("dfb_calc_batch_host_png", m)
        want[1] = want[1][:6] + (["o[%d]" % i for i in range(m)] or [None],) + want[1][7:]
        assert log(fake, f=fr, o=list(bufs)) == want


def test_calc_batch_png_refusals(e, fake):
    fr = gray(3)
    cap = png_cap(W, H)
    msg = r"^out: expected 2 C-contiguous uint8 buffers of at least %d bytes$" % cap
    for bad in ([np.zeros(cap, np.uint8)], [np.zeros(cap, np.uint8), np.zeros(cap - 1, np.uint8)],
                [np.zeros(cap, np.uint8), np.zeros(cap, np.int8)], [np.zeros(cap, np.uint8), np.zeros((2, cap), np.uint8)],
                [np.zeros(cap, np.uint8), np.zeros(2 * cap, np.uint8)[::2]], [np.zeros(cap, np.uint8), bytearray(cap)]):
        with pytest.raises(RuntimeError, match=msg):
            e.calc_batch_png(fr, 1, out=bad)
    assert set(c[0] for c in fake.calls) == {"dfb_png_max_bytes"}


def test_file_call_refusals(e, fake):
    fake.fail = {"dfb_process_bgr_batch_host": (_lib.DFB_ERR_INVALID_ARG, b"bound should > 0!")}
    with pytest.raises(RuntimeError, match="^bound should > 0!$"):
        e.process_bgr_batch(bgr(2), bound=0)
    fake.fail = {"dfb_extract_frames_jpeg_host": (_lib.DFB_ERR_CUDA, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb error -3$"):
        e.extract_frames_jpeg(jpegs(2))


# -- the list runner --

def stats_dict():
    return {"clips": 3, "flows": 5, "frames": 8, "seconds": 1.5, "workers": 2, "clips_per_worker": [1, 2], "flows_per_worker": [2, 3],
            "busy_seconds_per_worker": [0.25, 1.25], "finish_seconds_per_worker": [0.5, 1.5], "kernel_launches": 7, "h2d_bytes": 11,
            "d2h_bytes": 13}


@pytest.fixture
def runner(fake):
    r = listrun.ListRunner("farn", [0, 0, 1], 64, 48)
    (name, args), = fake.calls
    assert name == "dfb_list_open" and args[0] == b"farn" and list(args[1]) == [0, 0, 1] and args[2:5] == (3, 64, 48)
    assert desc(args[5], {}) == ("byref", "c_void_p") and desc(args[6], {}) == ("err", 512) and args[7] == 512
    fake.calls.clear()
    return r


def test_list_open_refusals(fake):
    fake.fail = {"dfb_list_open": (_lib.DFB_ERR_INVALID_ARG, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb_list_open failed \(-1\)$"):
        listrun.ListRunner("tvl1", [0], 64, 48)

    def refuse(alg, devs, ndev, mw, mh, out, err, err_len):
        err.value = b"unknown optical algorithm x"
        return _lib.DFB_ERR_UNKNOWN_ALGORITHM
    fake.on_dfb_list_open = refuse
    with pytest.raises(RuntimeError, match=r"^unknown optical algorithm x$"):
        listrun.ListRunner("x", [0], 64, 48)


def clips_of(sizes):
    return [gray(n, h, w, seed=n) for n, h, w in sizes]


@pytest.mark.parametrize("bound", [20, 0])
def test_list_run(runner, fake, bound):
    clips = clips_of([(3, 6, 8), (2, 4, 5)])
    got = []
    st = runner.run(clips, step=1, bound=bound, chunk_flows=4, on_chunk=lambda *a: got.append(
        a[:4] + tuple(None if v is None else [np.array(x) for x in v] for v in a[4:])))
    assert st == stats_dict()
    (name, args), = fake.calls
    assert name == "dfb_list_run" and args[0].value == 0x6000 and args[2:7] == (2, 1, bound, 4, None) and args[8] is None
    assert desc(args[9], {}) == ("byref", "ListStats") and desc(args[10], {}) == ("err", 512) and args[11] == 512
    arr = args[1]
    assert [(arr[k].n_frames, arr[k].height, arr[k].width) for k in range(2)] == [(3, 6, 8), (2, 4, 5)]
    assert [arr[0].frames[i] for i in range(3)] == [f.ctypes.data for f in clips[0]]
    for k, (clip, dev, first, last, qx, qy, flows) in enumerate(got):
        h, w = clips[k][0].shape
        m = len(clips[k]) - 1
        assert (clip, dev, first, last) == (k, 0, 0, True)
        if bound:
            assert flows is None and all(np.array_equal(qx[i], u8(i, 0, h, w)) and np.array_equal(qy[i], u8(i, 1, h, w)) for i in range(m))
        else:
            assert qx is None and qy is None and all(np.array_equal(flows[i], field(i, h, w)) for i in range(m))
    assert len(got) == 2
    # no callback, a queue, and a packed list
    packed = runner.pack(clips)
    q = type("Q", (), {"_q": 0x7000})()
    fake.calls.clear()
    assert runner.run(None, step=-2, bound=bound, queue=q, packed=packed) == stats_dict()
    (name, args), = fake.calls
    assert args[1] is packed[0] and args[2:9] == (2, -2, bound, 0, 0x7000, None, None)


def test_list_run_refusals(runner, fake):
    fake.fail = {"dfb_list_run": (_lib.DFB_ERR_CUDA, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb_list_run failed \(-3\)$"):
        runner.run(clips_of([(2, 4, 4)]))

    def refuse(r, clips, n, step, bound, chunk, queue, cb, user, st, err, err_len):
        err.value = b"clip 0: bound should > 0!"
        return _lib.DFB_ERR_INVALID_ARG
    fake.on_dfb_list_run = refuse
    with pytest.raises(RuntimeError, match=r"^clip 0: bound should > 0!$"):
        runner.run(clips_of([(2, 4, 4)]))
    with pytest.raises(RuntimeError, match=r"^clip 1: frames must be C-contiguous uint8 \[H,W\] images of one size$"):
        runner.run([gray(2), gray(2)[:1] + [gray(1, 4, 4)[0]]])


@pytest.mark.parametrize("save_type,step", [("jpg", 1), ("png", -1), ("h5", 2), ("jpg", 0)])
def test_list_run_videos(runner, fake, save_type, step):
    videos = [bgr(3), jpegs(4)]
    got = []
    st = runner.run_videos(videos, step=step, bound=15, save_type=save_type, quality=90, jpeg_exact=1, new_width=5, new_height=4,
                           new_short=0, chunk_flows=3, on_chunk=lambda *a: got.append(a))
    assert st == stats_dict()
    (name, args), = fake.calls
    assert name == "dfb_list_run_videos" and args[0].value == 0x6000 and args[2:13] == (2, step, 15, listrun._SAVE_TYPES[save_type], 90, 1, 5,
                                                                                  4, 0, 3, None)
    assert args[14] is None and desc(args[15], {}) == ("byref", "ListStats") and args[17] == 512
    assert fake.videos == [(_lib.VIDEO_BGR, 3, W, H), (_lib.VIDEO_JPEG, 4, 0, 0)]
    per = 2 if step != 0 and save_type != "png" else 1
    want = [(k, 1, 2, True, [file("list", j % per, j // per) for j in range(per * n)]) for k, n in enumerate([2, 3])]
    assert got == want
    fake.calls.clear()
    runner.run_videos(videos, save_type=save_type, queue=type("Q", (), {"_q": 0x7000})())
    (name, args), = fake.calls
    assert args[12:15] == (0x7000, None, None)


def test_list_run_videos_refusals(runner, fake):
    with pytest.raises(RuntimeError, match=r"^only jpg/png/h5 are supported \(no tif\) for output$"):
        runner.run_videos([bgr(2)], save_type="tif")
    with pytest.raises(RuntimeError, match=r"^video 1: frames must be uint8 \[H,W,3\] BGR images of one size, or JPEG files \(bytes\)$"):
        runner.run_videos([bgr(2), gray(2)])
    assert fake.calls == []
    fake.fail = {"dfb_list_run_videos": (_lib.DFB_ERR_CUDA, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb_list_run_videos failed \(-3\)$"):
        runner.run_videos([bgr(2)])


@pytest.mark.parametrize("fn", ["run_stream", "run_windows"])
@pytest.mark.parametrize("save_type,step", [("jpg", 1), ("png", 1), ("jpg", 0), ("h5", -1)])
def test_list_run_source(runner, fake, fn, save_type, step):
    videos = [bgr(3), jpegs(5)]
    reads, got = [], []

    def source(video, first, max_n):
        reads.append((video, first, max_n))
        return videos[video][first:first + max_n]
    st = getattr(runner, fn)(2, source, on_chunk=lambda *a: got.append(a), step=step, bound=12, save_type=save_type, quality=85,
                             jpeg_exact=1, new_width=0, new_height=0, new_short=4, chunk_flows=2)
    assert st == stats_dict()
    (name, args), = fake.calls
    assert name == "dfb_list_" + fn and args[0].value == 0x6000 and args[1] == 2
    assert args[3:13] == (step, 12, listrun._SAVE_TYPES[save_type], 85, 1, 0, 0, 4, 2, None) and args[14] is None
    assert desc(args[15], {}) == ("byref", "ListStats") and desc(args[16], {}) == ("err", 512) and args[17] == 512
    assert reads == [(0, 0, 4), (1, 0, 4)]
    assert fake.videos == [(_lib.VIDEO_BGR, 3, W, H), (_lib.VIDEO_JPEG, 4, 0, 0)]
    per = 2 if step != 0 and save_type != "png" else 1
    assert got == [(k, 1, 2, True, [file("list", j % per, j // per) for j in range(per * n)]) for k, n in enumerate([2, 3])]
    fake.calls.clear()
    assert getattr(runner, fn)(1, source, save_type=save_type, queue=type("Q", (), {"_q": 0x7000})()) == stats_dict()
    (name, args), = fake.calls
    assert args[12] == 0x7000


@pytest.mark.parametrize("fn", ["run_stream", "run_windows"])
def test_list_run_source_failures(runner, fake, fn):
    run = getattr(runner, fn)
    with pytest.raises(RuntimeError, match=r"^only jpg/png/h5 are supported \(no bmp\) for output$"):
        run(1, lambda *a: [], save_type="bmp")
    assert fake.calls == []

    def bad_source(video, first, max_n):
        if video == 1:
            raise ValueError("no such file")
        return bgr(2)
    with pytest.raises(RuntimeError, match=r"^video 1: no such file$"):
        run(2, bad_source)
    def silent(*a):
        raise LookupError()
    with pytest.raises(RuntimeError, match=r"^video 0: LookupError$"):
        run(1, silent)
    # the message is cut to the buffer the library gives (64 bytes here, with its terminating zero)
    with pytest.raises(RuntimeError, match=r"^video 0: frames must be uint8 \[H,W,3\] BGR images of one size, or JPEG fi$"):
        run(1, lambda *a: gray(2))

    def bad_chunk(*a):
        raise KeyError("on_chunk failed")
    # the failure is raised again; later windows are refused with the text of the stop
    with pytest.raises(KeyError, match="on_chunk failed"):
        run(2, lambda *a: bgr(2), on_chunk=bad_chunk)
    fake.fail = {"dfb_list_" + fn: (_lib.DFB_ERR_CUDA, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb_list_%s failed \(-3\)$" % fn):
        run(1, lambda *a: bgr(2))


def test_list_run_source_stops_after_failed_chunk(runner, fake):
    calls = []

    def bad_chunk(*a):
        calls.append(a[0])
        raise ValueError("disk full")
    with pytest.raises(ValueError, match="^disk full$"):
        runner.run_stream(3, lambda *a: bgr(2), on_chunk=bad_chunk)
    assert calls == [0]  # video 1's window is refused, so the run ends there (the fake returns the refusal)


@pytest.mark.parametrize("bound", [32, 0])
def test_run_list(fake, bound):
    clips = clips_of([(2, 4, 6), (4, 6, 8)])
    got = []
    st = listrun.run_list("tvl1", [1, 0], clips, step=2, bound=bound, chunk_flows=5,
                          on_chunk=lambda *a: got.append((a[0], a[4] is None, a[6] is None)))
    assert st == stats_dict()
    (name, args), = fake.calls
    assert name == "dfb_run_list" and args[0] == b"tvl1" and list(args[1]) == [1, 0] and args[2] == 2
    assert args[4:9] == (2, 2, bound, 5, None) and args[10] is None and desc(args[11], {}) == ("byref", "ListStats")
    assert desc(args[12], {}) == ("err", 512) and args[13] == 512
    assert [(args[3][k].n_frames, args[3][k].height, args[3][k].width) for k in range(2)] == [(2, 4, 6), (4, 6, 8)]
    assert got == [(0, not bound, bool(bound)), (1, not bound, bool(bound))]
    fake.calls.clear()
    fake.fail = {"dfb_run_list": (_lib.DFB_ERR_NO_DEVICE, b"")}
    with pytest.raises(RuntimeError, match=r"^dfb_run_list failed \(-6\)$"):
        listrun.run_list("tvl1", [0], clips)

    def refuse(*a):
        a[12].value = b"no CUDA device available"
        return _lib.DFB_ERR_NO_DEVICE
    fake.on_dfb_run_list = refuse
    with pytest.raises(RuntimeError, match=r"^no CUDA device available$"):
        listrun.run_list("tvl1", [0], clips)
