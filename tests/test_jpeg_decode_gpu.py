"""The GPU JPEG decoder (jpeg_decode.cu behind dfb_decode_jpeg_batch_device / dfb_process_jpeg_batch_host) against
cv2.imdecode: coefficients equal the restatement's (tests/jpeg_restate.py), pixels equal the golden fixture, the restatement
and live imdecode in both builds, and the `-if` flow chain gives process_bgr_batch's bytes on the imdecoded frames."""
import os

import cv2
import numpy as np
import pytest

import geometry_cases as G
import jpeg_cases as J
import jpeg_restate as R

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_decode_cases.npz")
_handles = {}


def handle(alg="tvl1", variant="default", size=(3840, 2160)):
    import denseflow_b200 as d
    key = (alg, variant, size)
    if key not in _handles:
        _handles[key] = d.create(alg, 0, size[0], size[1], variant=variant)
    return _handles[key]


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def decode(e, files, channels=3, **kw):
    import torch
    out = e.decode_jpeg_batch(files, channels, **kw)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def assert_pixels(e, files, want_bgr):
    got = decode(e, files, 3)
    gray = decode(e, files, 1)
    for i, (g, gg, w) in enumerate(zip(got, gray, want_bgr)):
        assert g.shape == w.shape, i
        assert np.array_equal(g, w), "frame %d: %d pixels differ" % (i, int((g != w).any(-1).sum()))
        assert np.array_equal(gg, cv2.cvtColor(w, cv2.COLOR_BGR2GRAY)), i


@pytest.mark.parametrize("case", ["small", "q100_noise", "restart", "optimized", "gray_q100_noise"])
def test_coefficients_equal_the_restatement(case):
    e = handle()
    b = {"small": J.encode(J.image("smooth", 17, 9), "420", 95),
         "q100_noise": J.encode(J.image("noise", 256, 340), "420", 100),  # long codes: thousands of subsequences
         "restart": J.encode(J.image("noise", 120, 200), "422", 97, restart=3),
         "optimized": J.encode(J.image("noise", 96, 96), "444", 90, optimize=True),
         "gray_q100_noise": J.encode(J.image("noise", 200, 300), "gray", 100)}[case]
    got, rounds = e.debug_jpeg_coefficients(b)
    want = R.coefficients(R.parse(b))
    assert got.shape == want.shape
    assert np.array_equal(got.astype(np.int64), want), "first differing block %d" % int(np.nonzero((got != want).any(1))[0][0])
    print("%s: %d blocks, %d sync rounds" % (case, len(got), rounds))
    # the rounds stop once no record changes; the longest segment's subsequence count (+1) bounds them.  Natural content
    # falls into step within the warm-up; i.i.d. noise at high quality (blocks without EOB) takes many rounds
    assert 1 <= rounds <= len(b) * 8 // 1024 + 2
    if case in ("small", "restart"):
        assert rounds <= 3


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_golden_fixture(variant):
    g = np.load(GOLDEN)
    n = int(g["n"])
    files = [g["jpg%d" % i].tobytes() for i in range(n)]
    assert_pixels(handle(variant=variant), files, [g["bgr%d" % i] for i in range(n)])


@pytest.mark.parametrize("variant", ["default", "strict"])
@pytest.mark.parametrize("sampling", J.SAMPLINGS)
def test_every_small_size_in_one_mixed_batch(variant, sampling):
    e = handle(variant=variant)
    files = [J.encode(J.image(k, h, w), sampling, q) for h in range(1, 18) for w in range(1, 18)
             for k, q in (("noise", 95), ("smooth", 50))]
    want = [imdecode(b) for b in files]
    for b, w in zip(files[::37], want[::37]):
        assert np.array_equal(R.decode(b), w)
    assert_pixels(e, files, want)


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_geometry_and_frame_sizes(variant):
    e = handle(variant=variant)
    sizes = G.SQUARES + G.STRIPS + [(340, 256), (1920, 1080), (2047, 1151), (3840, 2160)]
    for (w, h) in sizes:
        for samp in ("420", "422", "gray"):
            b = J.encode(J.image("smooth", h, w), samp, 95)
            assert_pixels(e, [b], [imdecode(b)])
    b = J.encode(J.image("smooth", 256, 340), "420", 95)
    assert np.array_equal(decode(e, [b])[0], R.decode(b))


def test_restarts_options_and_pillow_files():
    e = handle()
    files = [J.encode(J.image("noise", 45, 61), s, 95, restart=r) for s in J.SAMPLINGS for r in (1, 2, 7)]
    files += [J.encode(J.image("noise", 45, 61), s, 95, optimize=True) for s in J.SAMPLINGS]
    files += [J.encode(J.image("noise", 45, 61), s, 95, luma=90, chroma=30) for s in J.SAMPLINGS]
    files += list(J.pillow_files().values())
    files += [J.encode(J.image("noise", 1080, 1920), "420", 95, restart=1)]
    assert_pixels(e, files, [imdecode(b) for b in files])


def test_mixed_batch_equals_one_at_a_time():
    e = handle()
    files = [J.encode(J.image("noise", 70, 90), "420", 95), J.encode(J.image("smooth", 33, 17), "gray", 80),
             J.encode(J.image("smooth", 256, 340), "444", 95, restart=5), J.encode(J.image("noise", 9, 300), "440", 60)]
    batch = decode(e, files)
    for b, x in zip(files, batch):
        assert np.array_equal(decode(e, [b])[0], x)


def test_counts_inputs_outputs_and_streams():
    import torch
    e = handle()
    assert e.decode_jpeg_batch([]) == []
    files = [J.encode(J.image("noise", 31 + i, 45 + 2 * i), "420", 90) for i in range(6)]
    want = [imdecode(b) for b in files]
    # pinned input
    pinned = []
    for b in files:
        t = torch.empty(len(b), dtype=torch.uint8).pin_memory()
        t.numpy()[:] = np.frombuffer(b, np.uint8)
        pinned.append(t)
    for got, w in zip(decode(e, pinned), want):
        assert np.array_equal(got, w)
    # pitched output 1..3 bytes past a 64-byte row, on a non-default stream
    s = torch.cuda.Stream()
    for extra in (1, 2, 3):
        with torch.cuda.stream(s):
            out = e.decode_jpeg_batch(files, 3, max_width=64, max_height=64, pitch=64 * 3 + extra, stream=s.cuda_stream)
        s.synchronize()
        for o, w in zip(out, want):
            assert np.array_equal(o.cpu().numpy(), w)
    assert np.array_equal(decode(e, files[:1], 1)[0], cv2.cvtColor(want[0], cv2.COLOR_BGR2GRAY))


def test_refusals_then_a_good_call():
    from denseflow_b200 import _lib
    e = handle()
    good = J.encode(J.image("noise", 40, 40), "420", 90)
    for name, (b, kind, frag) in sorted(J.refusals().items()):
        with pytest.raises(RuntimeError, match=frag):
            e.decode_jpeg_batch([good, b])
        keep, ptrs, lens = e._jpeg_buffers([good, b])
        import torch
        out = torch.empty((2, 64, 192), dtype=torch.uint8, device="cuda")
        rc = e._L.dfb_decode_jpeg_batch_device(e._h, ptrs, lens, 2, 3, out.data_ptr(), 192, 64 * 192, 64, 64, None, None, None)
        assert rc == (_lib.DFB_ERR_UNSUPPORTED if kind == "unsupported" else _lib.DFB_ERR_INVALID_ARG), name
        assert b"frame 1" in e._L.dfb_last_error(e._h)
        assert np.array_equal(decode(e, [good])[0], imdecode(good))
    with pytest.raises(RuntimeError, match="does not fit"):
        e.decode_jpeg_batch([good], max_width=39, max_height=64)
    with pytest.raises(RuntimeError, match="channels"):
        e.decode_jpeg_batch([good], channels=2)


def test_frames_written_by_extract_frames():
    e = handle()
    frames = [J.image("smooth", 120, 160, seed=i) for i in range(3)] + [J.image("noise", 120, 160)]
    jpgs = e.extract_frames(frames) + e.extract_frames(frames, new_size=(75, 61))
    assert_pixels(e, jpgs, [imdecode(b) for b in jpgs])


def test_if_s0_composition():
    """-if -s=0: the frames decoded with channels 3, then dfb_encode_jpeg_bgr_device, equal encoding the imdecoded frames"""
    import torch
    e = handle()
    files = [J.encode(J.image("smooth", 90, 120, seed=i), "420", 95) for i in range(3)]
    for b, bgr in zip(files, e.decode_jpeg_batch(files, 3)):
        want = e.encode_jpeg_bgr_device(torch.from_numpy(imdecode(b)).cuda(), new_size=(60, 44))
        assert e.encode_jpeg_bgr_device(bgr, new_size=(60, 44)) == want


def _chain_frames(n, h, w, seed=0):
    from denseflow_b200 import synth
    gray = synth.stream(h, w, max(n, 1), seed=seed)[:n]
    return [J.encode(np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8), "420", 95) for g in gray]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("step", [1, -1, 3, -3])
@pytest.mark.parametrize("n_frames", [0, 1, 2, 9, 19])
def test_process_jpeg_batch_equals_bgr_chain(alg, step, n_frames):
    e = handle(alg, "default", (96, 64))
    files = _chain_frames(n_frames, 64, 96, seed=n_frames)
    bgr = [imdecode(b) for b in files]
    for new_size in (None, (72, 50)):
        got = e.process_jpeg_batch(files, step, 20, new_size)
        want = e.process_bgr_batch(bgr, step, 20, new_size) if bgr else []
        assert got == want
    # flow calls afterwards are unchanged
    from denseflow_b200 import synth
    a, b, _ = synth.pair(64, 96, 0)
    f1 = e.calc(a, b)
    e.process_jpeg_batch(files, step, 20)
    assert np.array_equal(e.calc(a, b), f1)


def test_process_jpeg_batch_1080p_groups():
    e = handle("tvl1", "default", (1920, 1080))
    files = _chain_frames(11, 1080, 1920, seed=5)
    bgr = [imdecode(b) for b in files]
    assert e.process_jpeg_batch(files, 1, 20) == e.process_bgr_batch(bgr, 1, 20)
    assert e.process_jpeg_batch(files[:6], 1, 20, (340, 256)) == e.process_bgr_batch(bgr[:6], 1, 20, (340, 256))


def test_process_jpeg_batch_refuses_mixed_sizes():
    e = handle("farn", "default", (96, 64))
    files = _chain_frames(3, 64, 96) + [J.encode(J.image("smooth", 64, 95), "420", 95)]
    with pytest.raises(RuntimeError, match="frame 3"):
        e.process_jpeg_batch(files, 1, 20)
