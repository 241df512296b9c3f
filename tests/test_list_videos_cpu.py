"""No-GPU checks of the host side of the video list: the size rule (dfb_new_size against get_new_size restated), the frame
size of a JPEG file (dfb_jpeg_info against imdecode) and the file names the reference gives a chunk's files."""
import ctypes as C
import itertools

import cv2
import numpy as np
import pytest

import jpeg_cases as J
from oracle import cv_restate

SIZES = [0, 1, 7, 255, 256, 257, 340]
SOURCES = [(1, 1), (340, 256), (256, 340), (1920, 1080), (1080, 1920), (455, 256)]


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from denseflow_b200 import _lib
    return _lib.load()


def _new_size(L, w, h, nw, nh, ns):
    dw, dh = C.c_int(-7), C.c_int(-7)
    rc = L.dfb_new_size(w, h, nw, nh, ns, C.byref(dw), C.byref(dh))
    return rc, (dw.value, dh.value)


def test_new_size_equals_get_new_size_over_the_grid(L):
    checked = 0
    for (w, h), nw, nh, ns in itertools.product(SOURCES, SIZES, SIZES, SIZES):
        if ns > 0 and nw + nh != 0:
            continue  # refused, below
        rc, got = _new_size(L, w, h, nw, nh, ns)
        assert rc == 0, (w, h, nw, nh, ns)
        do_resize, ww, hh = cv_restate.new_size(w, h, nw, nh, ns)
        assert got == (ww, hh), (w, h, nw, nh, ns)
        checked += 1
    assert checked == len(SOURCES) * (len(SIZES) ** 2 + len(SIZES) - 1)


@pytest.mark.parametrize("w,h", [(340, 256), (256, 340), (455, 256)])
def test_new_short_resizes_only_above_the_short_side(L, w, h):
    short = min(w, h)
    # min(w, h) == ns and ns + 1: no resize, the source size comes back
    for ns in (short, short + 1):
        assert _new_size(L, w, h, 0, 0, ns) == (0, (w, h))
    # ns - 1: the short side becomes ns, the long side (int)round(long / short * ns)
    rc, got = _new_size(L, w, h, 0, 0, short - 1)
    assert rc == 0 and got == cv_restate.new_size(w, h, 0, 0, short - 1)[1:] and min(got) == short - 1


def test_new_size_refusals_carry_the_reference_texts(L):
    from denseflow_b200 import _lib, api
    for args in [(-1, 0, 0), (0, -1, 0), (0, 0, -1)]:
        assert _new_size(L, 340, 256, *args)[0] == _lib.DFB_ERR_INVALID_ARG
        assert L.dfb_last_error(None) == b"height and width cannot < 0!"
    for args in [(256, 0, 256), (0, 256, 256), (340, 256, 1)]:
        assert _new_size(L, 340, 256, *args)[0] == _lib.DFB_ERR_INVALID_ARG
        assert L.dfb_last_error(None) == b"do not set height and width when set short!"
    with pytest.raises(RuntimeError, match="do not set height and width when set short!"):
        api.new_size(340, 256, new_width=10, new_short=10)
    assert api.new_size(340, 256, new_short=128) == (170, 128)


def _info(L, b):
    w, h = C.c_int(), C.c_int()
    rc = L.dfb_jpeg_info(b, len(b), C.byref(w), C.byref(h))
    return rc, (h.value, w.value)


@pytest.mark.parametrize("sampling", J.SAMPLINGS)
@pytest.mark.parametrize("h,w", [(1, 1), (7, 9), (16, 16), (37, 53), (256, 340), (255, 341)])
def test_jpeg_info_equals_imdecode(L, sampling, h, w):
    b = J.encode(J.image("smooth", h, w), sampling, 90)
    rc, hw = _info(L, b)
    assert rc == 0 and hw == cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR).shape[:2]


def test_jpeg_info_of_other_encoders(L):
    for name, b in J.pillow_files().items():
        rc, hw = _info(L, b)
        assert rc == 0 and hw == cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR).shape[:2], name


def test_jpeg_info_refusals(L):
    from denseflow_b200 import _lib
    for name, (b, kind, fragment) in J.refusals().items():
        rc, hw = _info(L, b)
        if kind == "unsupported":  # refused from the markers, as the decoder refuses it
            assert rc == _lib.DFB_ERR_UNSUPPORTED, name
            assert fragment in L.dfb_last_error(None).decode(), name
        else:  # the markers are sound; the decode finds the corrupt data
            assert rc == 0 and hw == (64, 64), name
    assert _info(L, b"not a jpeg file")[0] == _lib.DFB_ERR_INVALID_ARG
    assert b"no SOI marker" in L.dfb_last_error(None)
    full = J.encode(J.image("smooth", 40, 48), "420", 90)
    assert _info(L, full[:40])[0] == _lib.DFB_ERR_INVALID_ARG  # the file ends inside the headers


def _write_flow_images(prefix, step, start, n, ext):
    """writeFlowImages / writeFlowImagesPng (src/common.cpp:84-118), restated"""
    base = 0 if step > 0 else -step
    out = []
    for i in range(n):
        if step > 1:
            tmp = "_p%d_%05d.%s" % (step, start + i + base, ext)
        elif step < 0:
            tmp = "_m%d_%05d.%s" % (-step, start + i + base, ext)
        else:
            tmp = "_%05d.%s" % (start + i + base, ext)
        out.append(prefix + tmp)
    return out


@pytest.mark.parametrize("step", [1, 2, -1, -3])
@pytest.mark.parametrize("start,n", [(0, 4), (64, 3), (99998, 5)])
def test_output_names_equal_write_flow_images(step, start, n):
    from denseflow_b200.listrun import output_names
    xs = _write_flow_images("flow_x", step, start, n, "jpg")
    ys = _write_flow_images("flow_y", step, start, n, "jpg")
    assert output_names(step, start, n, "jpg") == [f for pair in zip(xs, ys) for f in pair]
    assert output_names(step, start, n, "png") == _write_flow_images("flow", step, start, n, "png")


def test_output_names_of_extracted_frames():
    from denseflow_b200.listrun import output_names
    # writeImages (src/common.cpp:73-82) with the "img" prefix (src/denseflow_gpu.cpp:95)
    assert output_names(0, 8, 3) == ["img_00008.jpg", "img_00009.jpg", "img_00010.jpg"]
    assert output_names(0, 0, 0, "png") == []
