"""Byte and pair counters of the batched host pipelines and the single-image encoders, in both settings of "jpeg_exact".
Every batched call runs at least three groups, so each group's read-back overlaps the next group's encode: the
counters must follow from the shapes and the returned lengths alone."""
import numpy as np
import pytest

from denseflow_b200 import synth

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

W, H = 64, 48
N = 20  # 19 pairs: three groups of at most 8 (Farneback's batch) in the flow pipelines, three groups of 8 frames in extraction


@pytest.fixture(scope="module")
def gray():
    a, b, _ = synth.pair(H, W, 7)
    return [np.roll(a, i, 1) if i % 2 else np.roll(b, i, 0) for i in range(N)]


@pytest.fixture(scope="module")
def bgr(gray):
    return [np.stack([g, np.roll(g, 3, 1), 255 - g], -1).astype(np.uint8) for g in gray]


def _handle(exact):
    import denseflow_b200 as d
    e = d.FarnebackOpticalFlow.create(0, 128, 96)
    e.set("jpeg_exact", exact)
    return e


def _delta(e, call):
    before = e.counters()
    out = call()
    after = e.counters()
    return out, {k: after[k] - before[k] for k in ("d2h_bytes", "h2d_bytes", "pairs")}


def _pinned(shape):
    import torch
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True).numpy()


@pytest.mark.parametrize("pinned", [False, True])
def test_calc_batch_host_counters(gray, pinned):
    import torch
    e = _handle(0)
    m = N - 1
    flows = torch.empty((m, H, W, 2), dtype=torch.float32, pin_memory=True).numpy() if pinned else None
    _, c = _delta(e, lambda: e.calc_batch(gray, flows=flows))
    assert c == {"d2h_bytes": m * W * H * 8, "h2d_bytes": N * W * H, "pairs": m}

    if pinned:
        qx, qy = _pinned((m, H, W)), _pinned((m, H, W))
        _, c = _delta(e, lambda: e.calc_batch_u8_into(gray, 1, 20, qx, qy))
    else:
        _, c = _delta(e, lambda: e.calc_batch(gray, bound=20))
    assert c == {"d2h_bytes": m * W * H * 2, "h2d_bytes": N * W * H, "pairs": m}

    cap = e._L.dfb_png_max_bytes(W, H)
    out = [_pinned((cap,)) for _ in range(m)] if pinned else None
    files, c = _delta(e, lambda: e.calc_batch_png(gray, out=out))
    assert len(files) == m
    assert c == {"d2h_bytes": sum(len(f) for f in files), "h2d_bytes": N * W * H, "pairs": m}


@pytest.mark.parametrize("exact", [0, 1])
def test_flow_chain_counters(bgr, exact):
    e = _handle(exact)
    m = N - 1
    for size in (None, (48, 32)):
        pairs, c = _delta(e, lambda: e.process_bgr_batch(bgr, new_size=size))
        assert len(pairs) == m
        assert c == {"d2h_bytes": sum(len(x) + len(y) for x, y in pairs), "h2d_bytes": N * W * H * 3, "pairs": m}, size

    jpegs = [cv2.imencode(".jpg", f)[1].tobytes() for f in bgr]
    pairs, c = _delta(e, lambda: e.process_jpeg_batch(jpegs))
    assert len(pairs) == m
    assert c == {"d2h_bytes": sum(len(x) + len(y) for x, y in pairs), "h2d_bytes": sum(len(j) for j in jpegs), "pairs": m}


@pytest.mark.parametrize("exact", [0, 1])
def test_extract_frames_counters(bgr, exact):
    e = _handle(exact)
    for size in (None, (40, 30)):
        files, c = _delta(e, lambda: e.extract_frames(bgr, size))
        assert len(files) == N
        assert c == {"d2h_bytes": sum(len(f) for f in files), "h2d_bytes": N * W * H * 3, "pairs": 0}, size


@pytest.mark.parametrize("exact", [0, 1])
def test_single_image_encoder_counters(gray, bgr, exact):
    """each single-image encoder counts its file's bytes, whichever JPEG encoder the handle uses"""
    import torch
    e = _handle(exact)
    plane = torch.from_numpy(gray[0]).cuda()
    image = torch.from_numpy(bgr[0]).cuda()
    for call in (lambda: e.encode_jpeg_gray_device(plane), lambda: e.encode_jpeg_bgr_device(image),
                 lambda: e.encode_jpeg_bgr_device(image, (40, 30)), lambda: e.encode_png_bgr_device(image)):
        f, c = _delta(e, call)
        assert len(f) > 0
        assert c == {"d2h_bytes": len(f), "h2d_bytes": 0, "pairs": 0}
