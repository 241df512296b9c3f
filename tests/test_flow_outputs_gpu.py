"""The outputs of the host flow calls through the C ABI.

- Refusals: every host flow batch entry point returns the same code and the same dfb_last_error text for a missing output
  array, a null or device per-pair pointer, use_initial_flow on a call that has no float buffer to read a start from, and
  inputs that break two checks at once (which one wins is part of the contract).
- Page-locked and pageable outputs in one call: pairs whose buffers are all page-locked are read back directly, the others
  through pinned staging; the bytes and the h2d / d2h counts equal those of an all-pageable call, warm-started or not."""
import ctypes as C

import numpy as np
import pytest

import denseflow_b200 as d
from denseflow_b200 import _lib, synth

pytestmark = pytest.mark.gpu

W, H = 64, 48
N = 3  # frames of the refusal calls: pairs 0 and 1 with step 1
INVALID, SIZE = _lib.DFB_ERR_INVALID_ARG, _lib.DFB_ERR_SIZE

SUFFIX = ": use_initial_flow is set, so the flow buffer must hold the initial flow"
REFUSED = ("use_initial_flow is set: only the calls that take a float flow buffer (dfb_calc_device / _host / _batch_host / "
           "_batch_device and their _planes forms) read an initial flow; set it to 0 for this call")


def _pair_msg(label, j):
    return "%s %d is null or a device pointer (host entry point)" % (label, j)


def _frames_msg(j):
    return "frames[%d] is null or a device pointer (host entry point: use dfb_calc_batch_device)" % j


def _bgr_msg(j):
    return "bgr[%d] is null or a device pointer (host entry point)" % j


class _Env:
    """One handle, valid inputs and outputs for every entry point, and a device buffer to pass where host memory is due."""

    def __init__(self):
        import cv2
        import torch
        self.e = d.create("tvl1", 0, W, H)
        self.L, self.h = self.e._L, self.e._h
        self.gray = synth.stream(H, W, N, 0)
        self.bgr = np.ascontiguousarray(np.repeat(self.gray[..., None], 3, -1))
        self.jpeg = [np.frombuffer(cv2.imencode(".jpg", f)[1].tobytes(), np.uint8) for f in self.bgr]
        self.dev = torch.zeros(W * H * 8, dtype=torch.uint8, device="cuda")
        self.cap = max(self.L.dfb_jpeg_max_bytes(W, H), self.L.dfb_png_max_bytes(W, H))
        M = N - 1
        self.field = [np.zeros((H, W, 2), np.float32) for _ in range(M)]
        self.fx = [np.zeros((H, W), np.float32) for _ in range(M)]
        self.fy = [np.zeros((H, W), np.float32) for _ in range(M)]
        self.qx = [np.zeros((H, W), np.uint8) for _ in range(M)]
        self.qy = [np.zeros((H, W), np.uint8) for _ in range(M)]
        self.files = [np.zeros(self.cap, np.uint8) for _ in range(M)]
        self.files_y = [np.zeros(self.cap, np.uint8) for _ in range(M)]
        self.len_x, self.len_y = (C.c_size_t * M)(), (C.c_size_t * M)()

    def ptrs(self, bufs, bad=None):
        """Pointer array of bufs; bad = {j: "null" | "dev"} replaces pair j's pointer."""
        p = [b.ctypes.data for b in bufs]
        for j, what in (bad or {}).items():
            p[j] = None if what == "null" else self.dev.data_ptr()
        return (C.c_void_p * len(p))(*p)


def _arr(env, o, key, bufs):
    """o[key]: absent -> the valid array of bufs, None -> a null array, a dict -> bufs with pairs replaced (see _Env.ptrs)."""
    if key not in o:
        return env.ptrs(bufs)
    return None if o[key] is None else env.ptrs(bufs, o[key])


def _call(env, entry, **o):
    L, h = env.L, env.h
    n, step = o.get("n", N), o.get("step", 1)
    w, hh = o.get("w", W), o.get("hh", H)
    frames = _arr(env, o, "frames", env.gray)
    bgr = _arr(env, o, "bgr", env.bgr)
    jp = _arr(env, o, "jpeg", env.jpeg)
    jl = (C.c_size_t * N)(*[len(j) for j in env.jpeg])
    dw, dh = o.get("dw", 0), o.get("dh", 0)
    bound, cap = o.get("bound", 20), env.cap
    lx = env.len_x if o.get("lx", True) else None
    ly = env.len_y if o.get("ly", True) else None
    if entry == "dfb_calc_host":
        dev = env.dev.data_ptr()
        ab = {"null": None, "dev": dev}
        a = ab[o["a"]] if "a" in o else env.gray[0].ctypes.data
        flow = ab[o["flow"]] if "flow" in o else env.field[0].ctypes.data
        return L.dfb_calc_host(h, a, env.gray[1].ctypes.data, w, hh, flow)
    if entry == "dfb_calc_batch_host":
        return L.dfb_calc_batch_host(h, frames, n, step, w, hh, _arr(env, o, "x", env.field))
    if entry == "dfb_calc_batch_host_u8":
        return L.dfb_calc_batch_host_u8(h, frames, n, step, w, hh, bound, _arr(env, o, "x", env.qx), _arr(env, o, "y", env.qy))
    if entry == "dfb_calc_batch_host_planes":
        return L.dfb_calc_batch_host_planes(h, frames, n, step, w, hh, _arr(env, o, "x", env.fx), _arr(env, o, "y", env.fy))
    if entry == "dfb_calc_batch_host_png":
        return L.dfb_calc_batch_host_png(h, frames, n, step, w, hh, _arr(env, o, "x", env.files), cap, lx)
    jpg = (bound, 95, _arr(env, o, "x", env.files), _arr(env, o, "y", env.files_y), cap, lx, ly)
    png = (_arr(env, o, "x", env.files), cap, lx)
    planes = (_arr(env, o, "x", env.fx), _arr(env, o, "y", env.fy))
    if entry == "dfb_process_bgr_batch_host":
        return L.dfb_process_bgr_batch_host(h, bgr, n, step, W, H, dw, dh, *jpg)
    if entry == "dfb_process_bgr_batch_host_png":
        return L.dfb_process_bgr_batch_host_png(h, bgr, n, step, W, H, dw, dh, *png)
    if entry == "dfb_process_bgr_batch_host_planes":
        return L.dfb_process_bgr_batch_host_planes(h, bgr, n, step, W, H, dw, dh, *planes)
    if entry == "dfb_process_jpeg_batch_host":
        return L.dfb_process_jpeg_batch_host(h, jp, jl, n, step, dw, dh, *jpg)
    if entry == "dfb_process_jpeg_batch_host_png":
        return L.dfb_process_jpeg_batch_host_png(h, jp, jl, n, step, dw, dh, *png)
    if entry == "dfb_process_jpeg_batch_host_planes":
        return L.dfb_process_jpeg_batch_host_planes(h, jp, jl, n, step, dw, dh, *planes)
    raise AssertionError(entry)


# (entry point, use_initial_flow, arguments changed from a valid call, return code, dfb_last_error text)
CASES = [
    # dfb_calc_host: a float2 field, which may hold the initial flow
    ("dfb_calc_host", 0, {"flow": "null"}, INVALID, "null buffer"),
    ("dfb_calc_host", 1, {"flow": "null"}, INVALID, "null buffer" + SUFFIX),
    ("dfb_calc_host", 0, {"flow": "dev"}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_host", 1, {"flow": "dev"}, INVALID, _pair_msg("output", 0) + SUFFIX),
    ("dfb_calc_host", 0, {"a": "null"}, INVALID, "null buffer"),
    ("dfb_calc_host", 0, {"a": "dev", "flow": "dev"}, INVALID, _frames_msg(0)),
    ("dfb_calc_host", 0, {"w": 0, "flow": "dev"}, INVALID, "width/height must be positive"),
    # dfb_calc_batch_host
    ("dfb_calc_batch_host", 0, {"x": None}, INVALID, "flows is null"),
    ("dfb_calc_batch_host", 1, {"x": None}, INVALID, "flows is null" + SUFFIX),
    ("dfb_calc_batch_host", 0, {"x": {1: "null"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host", 1, {"x": {1: "null"}}, INVALID, _pair_msg("output", 1) + SUFFIX),
    ("dfb_calc_batch_host", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host", 0, {"x": None, "step": 0}, INVALID, "flows is null"),
    ("dfb_calc_batch_host", 0, {"x": {0: "null"}, "frames": {1: "dev"}}, INVALID, _frames_msg(1)),
    ("dfb_calc_batch_host", 0, {"x": {0: "null"}, "w": W + 1}, SIZE, "frame 65x48 exceeds the 64x48 given to dfb_create"),
    ("dfb_calc_batch_host", 0, {"x": None, "n": 1}, 0, None),
    # dfb_calc_batch_host_u8: no float buffer, so no initial flow
    ("dfb_calc_batch_host_u8", 1, {}, INVALID, REFUSED),
    ("dfb_calc_batch_host_u8", 0, {"x": None}, INVALID, "qx/qy is null"),
    ("dfb_calc_batch_host_u8", 0, {"y": None}, INVALID, "qx/qy is null"),
    ("dfb_calc_batch_host_u8", 0, {"x": {1: "null"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host_u8", 0, {"y": {0: "null"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host_u8", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host_u8", 0, {"y": {1: "dev"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host_u8", 1, {"bound": 0}, INVALID, REFUSED),
    ("dfb_calc_batch_host_u8", 0, {"bound": 0, "x": None}, INVALID, "bound should > 0!"),
    ("dfb_calc_batch_host_u8", 0, {"y": {0: "null"}, "frames": None}, INVALID, "frames is null"),
    # dfb_calc_batch_host_planes: two float planes, which may hold the initial flow
    ("dfb_calc_batch_host_planes", 0, {"x": None}, INVALID, "fx/fy is null"),
    ("dfb_calc_batch_host_planes", 1, {"y": None}, INVALID, "fx/fy is null" + SUFFIX),
    ("dfb_calc_batch_host_planes", 0, {"x": {0: "null"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host_planes", 0, {"y": {1: "null"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host_planes", 1, {"y": {1: "null"}}, INVALID, _pair_msg("output", 1) + SUFFIX),
    ("dfb_calc_batch_host_planes", 0, {"x": {1: "dev"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host_planes", 0, {"y": {0: "dev"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host_planes", 0, {"x": None, "w": 0}, INVALID, "fx/fy is null"),
    ("dfb_calc_batch_host_planes", 0, {"y": {0: "null"}, "step": 0}, INVALID, "step must be non-zero for flow extraction"),
    # dfb_calc_batch_host_png
    ("dfb_calc_batch_host_png", 1, {}, INVALID, REFUSED),
    ("dfb_calc_batch_host_png", 0, {"x": None}, INVALID, "png / len is null"),
    ("dfb_calc_batch_host_png", 0, {"lx": False}, INVALID, "png / len is null"),
    ("dfb_calc_batch_host_png", 0, {"x": {1: "null"}}, INVALID, _pair_msg("output", 1)),
    ("dfb_calc_batch_host_png", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("output", 0)),
    ("dfb_calc_batch_host_png", 1, {"x": None}, INVALID, REFUSED),
    ("dfb_calc_batch_host_png", 0, {"x": {0: "null"}, "frames": {0: "null"}}, INVALID, _frames_msg(0)),
    # dfb_process_bgr_batch_host: two JPEG files per pair
    ("dfb_process_bgr_batch_host", 1, {}, INVALID, REFUSED),
    ("dfb_process_bgr_batch_host", 0, {"x": None}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host", 0, {"y": None}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host", 0, {"lx": False}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host", 0, {"ly": False}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host", 0, {"x": {1: "null"}}, INVALID, _pair_msg("jpeg output", 1)),
    ("dfb_process_bgr_batch_host", 0, {"y": {0: "null"}}, INVALID, _pair_msg("jpeg output", 0)),
    ("dfb_process_bgr_batch_host", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("jpeg output", 0)),
    ("dfb_process_bgr_batch_host", 0, {"y": {1: "dev"}}, INVALID, _pair_msg("jpeg output", 1)),
    ("dfb_process_bgr_batch_host", 1, {"bound": 0}, INVALID, REFUSED),
    ("dfb_process_bgr_batch_host", 0, {"bound": 0, "x": None}, INVALID, "bound should > 0!"),
    ("dfb_process_bgr_batch_host", 0, {"x": None, "bgr": {1: "null"}}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host", 0, {"x": {0: "null"}, "bgr": {1: "dev"}}, INVALID, _bgr_msg(1)),
    ("dfb_process_bgr_batch_host", 0, {"x": None, "n": 1}, 0, None),
    # dfb_process_bgr_batch_host_png
    ("dfb_process_bgr_batch_host_png", 1, {}, INVALID, REFUSED),
    ("dfb_process_bgr_batch_host_png", 0, {"x": None}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host_png", 0, {"lx": False}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host_png", 0, {"x": {1: "null"}}, INVALID, _pair_msg("png output", 1)),
    ("dfb_process_bgr_batch_host_png", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("png output", 0)),
    ("dfb_process_bgr_batch_host_png", 0, {"x": None, "dw": -1}, INVALID, "bad geometry"),
    # dfb_process_bgr_batch_host_planes: float planes, but the chains read no initial flow
    ("dfb_process_bgr_batch_host_planes", 1, {}, INVALID, REFUSED),
    ("dfb_process_bgr_batch_host_planes", 0, {"x": None}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host_planes", 0, {"y": None}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host_planes", 0, {"x": {0: "null"}}, INVALID, _pair_msg("plane output", 0)),
    ("dfb_process_bgr_batch_host_planes", 0, {"y": {1: "null"}}, INVALID, _pair_msg("plane output", 1)),
    ("dfb_process_bgr_batch_host_planes", 0, {"y": {0: "dev"}}, INVALID, _pair_msg("plane output", 0)),
    ("dfb_process_bgr_batch_host_planes", 1, {"x": None}, INVALID, REFUSED),
    ("dfb_process_bgr_batch_host_planes", 0, {"y": None, "bgr": {0: "dev"}}, INVALID, "null output"),
    ("dfb_process_bgr_batch_host_planes", 0, {"x": {1: "dev"}, "bgr": {2: "null"}}, INVALID, _bgr_msg(2)),
    # dfb_process_jpeg_batch_host: the JPEG files are parsed before the outputs are checked
    ("dfb_process_jpeg_batch_host", 1, {}, INVALID, REFUSED),
    ("dfb_process_jpeg_batch_host", 0, {"x": None}, INVALID, "null output"),
    ("dfb_process_jpeg_batch_host", 0, {"ly": False}, INVALID, "null output"),
    ("dfb_process_jpeg_batch_host", 0, {"x": {0: "null"}}, INVALID, _pair_msg("jpeg output", 0)),
    ("dfb_process_jpeg_batch_host", 0, {"y": {1: "null"}}, INVALID, _pair_msg("jpeg output", 1)),
    ("dfb_process_jpeg_batch_host", 0, {"y": {0: "dev"}}, INVALID, _pair_msg("jpeg output", 0)),
    ("dfb_process_jpeg_batch_host", 0, {"bound": -1, "y": None}, INVALID, "bound should > 0!"),
    ("dfb_process_jpeg_batch_host", 0, {"x": None, "jpeg": {1: "null"}}, INVALID, "frame 1: null or empty JPEG buffer"),
    ("dfb_process_jpeg_batch_host", 0, {"x": None, "dw": W + 1, "dh": H}, SIZE, "frame 65x48 exceeds the 64x48 given to dfb_create"),
    # dfb_process_jpeg_batch_host_png
    ("dfb_process_jpeg_batch_host_png", 1, {}, INVALID, REFUSED),
    ("dfb_process_jpeg_batch_host_png", 0, {"x": None}, INVALID, "null output"),
    ("dfb_process_jpeg_batch_host_png", 0, {"lx": False}, INVALID, "null output"),
    ("dfb_process_jpeg_batch_host_png", 0, {"x": {1: "null"}}, INVALID, _pair_msg("png output", 1)),
    ("dfb_process_jpeg_batch_host_png", 0, {"x": {1: "dev"}}, INVALID, _pair_msg("png output", 1)),
    ("dfb_process_jpeg_batch_host_png", 0, {"x": None, "step": 0}, INVALID, "step must be non-zero for flow extraction"),
    ("dfb_process_jpeg_batch_host_png", 0, {"x": {0: "null"}, "jpeg": {0: "dev"}}, INVALID,
     "frame 0: the JPEG bytes must be in host memory"),
    # dfb_process_jpeg_batch_host_planes
    ("dfb_process_jpeg_batch_host_planes", 1, {}, INVALID, REFUSED),
    ("dfb_process_jpeg_batch_host_planes", 0, {"y": None}, INVALID, "null output"),
    ("dfb_process_jpeg_batch_host_planes", 0, {"x": {1: "null"}}, INVALID, _pair_msg("plane output", 1)),
    ("dfb_process_jpeg_batch_host_planes", 0, {"y": {0: "null"}}, INVALID, _pair_msg("plane output", 0)),
    ("dfb_process_jpeg_batch_host_planes", 0, {"x": {0: "dev"}}, INVALID, _pair_msg("plane output", 0)),
    ("dfb_process_jpeg_batch_host_planes", 1, {"frames": None, "jpeg": None}, INVALID, REFUSED),
    ("dfb_process_jpeg_batch_host_planes", 0, {"x": None, "jpeg": None}, INVALID, "frames is null"),
]


@pytest.fixture(scope="module")
def env():
    v = _Env()
    yield v
    v.e.release()


@pytest.mark.parametrize("entry,init,args,rc,text", CASES)
def test_refusals(env, entry, init, args, rc, text):
    env.e.set("use_initial_flow", init)
    before = env.e.counters()
    try:
        assert _call(env, entry, **args) == rc
    finally:
        env.e.set("use_initial_flow", 0)
    if text is not None:
        assert env.L.dfb_last_error(env.h).decode() == text
    after = env.e.counters()
    assert (after["pairs"], after["h2d_bytes"], after["d2h_bytes"]) == (before["pairs"], before["h2d_bytes"], before["d2h_bytes"])


# ---- page-locked and pageable outputs in one call ----

LANES = 3          # pairs per group: output slots hold 3 pairs each
M = 4 * LANES + 1  # five groups: each of the two output slots is used at least twice
BOUND = 8


def _pinned(shape, dtype):
    import torch
    t = torch.empty(shape, dtype={np.float32: torch.float32, np.uint8: torch.uint8}[dtype], pin_memory=True)
    return t.numpy()


def _mixed_buffers(shape, dtype, k):
    """k buffers per pair for M pairs: pair j's are page-locked, pageable, or (k = 2) a page-locked x with a pageable y, in a
    pattern that moves across the pairs' positions in their groups."""
    out = [[None] * M for _ in range(k)]
    for j in range(M):
        kind = (j + j // LANES) % 3
        for c in range(k):
            pinned = kind == 0 or (kind == 2 and c == 0 and k == 2)
            out[c][j] = _pinned(shape, dtype) if pinned else np.empty(shape, dtype)
    return out


LAYOUTS = {
    # layout: (entry point, k buffers per pair, shape, dtype)
    "field": ("dfb_calc_batch_host", 1, (H, W, 2), np.float32),
    "u8": ("dfb_calc_batch_host_u8", 2, (H, W), np.uint8),
    "planes": ("dfb_calc_batch_host_planes", 2, (H, W), np.float32),
}


def _starts(layout):
    """Each pair's initial flow, a different one per pair, in the layout's buffers."""
    rng = np.random.default_rng(7)
    f = (rng.standard_normal((M, H, W, 2)) * 1.5).astype(np.float32)
    return [[f[j]] for j in range(M)] if layout == "field" else [[f[j, ..., 0].copy(), f[j, ..., 1].copy()] for j in range(M)]


def _run(e, layout, frames, bufs):
    L = e._L
    entry, k = LAYOUTS[layout][:2]
    fp = (C.c_void_p * len(frames))(*[f.ctypes.data for f in frames])
    ptrs = [(C.c_void_p * M)(*[b.ctypes.data for b in bufs[c]]) for c in range(k)]
    e.reset_counters()
    args = (BOUND,) if layout == "u8" else ()
    assert getattr(L, entry)(e._h, fp, M + 1, 1, W, H, *args, *ptrs) == 0, L.dfb_last_error(e._h)
    c = e.counters()
    return b"".join(b.tobytes() for c_ in range(k) for b in bufs[c_]), (c["pairs"], c["h2d_bytes"], c["d2h_bytes"])


@pytest.mark.parametrize("layout,init", [("field", 0), ("u8", 0), ("planes", 0), ("field", 1), ("planes", 1)])
def test_mixed_pinned_and_pageable_outputs(layout, init):
    entry, k, shape, dtype = LAYOUTS[layout]
    e = d.create("tvl1", 0, W, H)
    e.set("lanes", LANES)
    e.set("use_initial_flow", init)
    frames = list(synth.stream(H, W, M + 1, 3))
    pageable = [[np.empty(shape, dtype) for _ in range(M)] for _ in range(k)]
    mixed = _mixed_buffers(shape, dtype, k)
    if init:
        starts = _starts(layout)
        for bufs in (pageable, mixed):
            for j in range(M):
                for c in range(k):
                    bufs[c][j][...] = starts[j][c]
    want, want_counts = _run(e, layout, frames, pageable)
    got, got_counts = _run(e, layout, frames, mixed)
    assert got_counts == want_counts and want_counts[0] == M
    assert got == want
    if init:  # the starts were read: a cold call gives other flows
        e.set("use_initial_flow", 0)
        cold, _ = _run(e, layout, frames, [[np.empty(shape, dtype) for _ in range(M)] for _ in range(k)])
        assert cold != want
    e.release()
