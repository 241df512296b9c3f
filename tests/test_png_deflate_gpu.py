"""The GPU PNG encoder (denseflow_b200/csrc/png_encode.cu) on content built to reach zlib's deflate edges
(tests/deflate_cases.py, each checked to reach its edge in tests/test_png_deflate_cpu.py): byte for byte the restatement
(tests/png_restate.py, pinned to cv2.imencode), alone, in batches through one encoder call, and on a realistic packed flow."""
import numpy as np
import pytest

import deflate_cases as D
import inflate_trace as T
import png_cases as PC
import png_restate as P
import zlib_sizes as Z
from oracle import cv_restate as R

pytestmark = pytest.mark.gpu

_handles = {}
_cases = {}


def handle(variant="default", size=(3840, 2160)):
    import denseflow_b200 as d
    key = (variant, size)
    if key not in _handles:
        _handles[key] = d.create("tvl1", 0, size[0], size[1], variant=variant)
    return _handles[key]


def handle_for(img, variant="default"):
    """the default handle, or a short wide one for the one-row cases wider than 3840"""
    h, w = img.shape[:2]
    return handle(variant) if w <= 3840 and h <= 2160 else handle(variant, (16384, 16))


def cases():
    if not _cases:
        _cases.update((n, img) for n, img, _ in D.cases())
    return _cases


NAMES = [n for n, _, _ in D.cases()]


def _same(got, want, what):
    assert got == want, (what, len(got), len(want), T.first_difference(P.idat_stream(got), P.idat_stream(want)))


def encode(e, img):
    import torch
    return e.encode_png_bgr_device(torch.from_numpy(np.ascontiguousarray(img)).cuda())


def encode_batch(e, imgs):
    """the images (one size) through one call of the batch encoder -st=png uses: the "png_encode_batch" debug stage"""
    n = len(imgs)
    h, w = imgs[0].shape[:2]
    stack = np.concatenate(imgs, 0)
    cap = e._L.dfb_png_max_bytes(w, h)
    (files,), lens = e.debug_run_kernel("png_encode_batch", [stack[..., c] for c in range(3)], 1, scalars=(n,),
                                        out_shape=(n, cap), all_scalars=True)
    return [files[i, :int(lens[i])].astype(np.uint8).tobytes() for i in range(n)]


@pytest.mark.parametrize("variant", ["default", "strict"])
@pytest.mark.parametrize("name", NAMES)
def test_case_equals_imencode(name, variant):
    import cv2
    img = cases()[name]
    got = encode(handle_for(img, variant), img)
    _same(got, P.encode(img), name)
    assert np.array_equal(cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_COLOR), img)


def _noise_like(img, seed):
    h, w = img.shape[:2]
    return PC.image("noise", h, w, seed=seed)


# one batch per image size: the edge cases at positions >= 1, between noise images of the same size
BATCHED = ["fibonacci17", "lucas19","deep_middle_block", "deep_with_lengths", "geometric0", "stored+4", "fixed=dynamic+0",
           "flush_at_run_match", "idat_8192", "idat_8193", "idat_16384", "window_2^12 w1"]


@pytest.mark.parametrize("name", BATCHED)
def test_batch_equals_single(name):
    img = cases()[name]
    e = handle_for(img)
    others = [c for n, c in cases().items() if c.shape == img.shape and n != name]
    imgs = [_noise_like(img, 1), img, _noise_like(img, 2)] + others[:2] + [img]
    got = encode_batch(e, imgs)
    for i, (g, x) in enumerate(zip(got, imgs)):
        _same(g, P.encode(x), (name, i))
        _same(g, encode(e, x), (name, i, "single"))


def test_batch_of_one_and_sixteen():
    e = handle()
    img = cases()["idat_8192"]
    assert encode_batch(e, [img]) == [P.encode(img)]
    imgs = [cases()["idat_%d" % t] for t in (8191, 8192, 8193)] * 5 + [_noise_like(img, 3)]
    assert encode_batch(e, imgs) == [P.encode(x) for x in imgs]


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_realistic_flow_at_1080p(variant):
    """a packed 1920 x 1080 flow field whose zlib stream has blocks that need the literal-tree repair, packed on the GPU,
    encoded alone and in a batch with a noise image"""
    import torch
    e = handle(variant)
    flow = D.synthetic_flow()
    img, bx, by = R.flow_to_png_image(flow)
    assert any(b["type"] == "dynamic" and b["lit"]["overflow"] for b in Z.blocks(P.scanlines(img)))
    bgr, bounds = e.flow_to_png_image_device(torch.from_numpy(flow).cuda())
    torch.cuda.synchronize()
    assert bounds == (bx, by) and np.array_equal(bgr.cpu().numpy(), img)
    want = P.encode(img)
    _same(e.encode_png_bgr_device(bgr), want, "single")
    got = encode_batch(e, [_noise_like(img, 4), img])
    _same(got[1], want, "batch")
    _same(got[0], P.encode(_noise_like(img, 4)), "batch noise")
