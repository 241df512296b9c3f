"""The nvJPEG files (handle parameter "jpeg_exact" = 0, the default) at sizes with a partial 8 x 8 block or 16 x 16 MCU.

nvJPEG reads whole blocks (gray) or MCUs (colour) from the planes it is handed, so the bytes past the image must be the
padding libjpeg would code there, and nothing else.  Three things are held here:
  - a file is a function of the image alone: the same whatever lies around the caller's plane, whatever a handle's scratch
    held before, and whichever list worker wrote it;
  - the padded planes nvJPEG gets are libjpeg's (the "jpeg_padded_*" debug stages against tests/ycc_restate.py and the
    padding rules of tests/jpeg_encode_restate.py), bit for bit;
  - decoded, every 8 x 8 block and the last block row and column are as close to the image as imencode's round trip.
nvJPEG's bytes depend on the library version, so no file is kept as a golden: every comparison is made within one run."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

from denseflow_b200 import synth  # noqa: E402

import jpeg_encode_restate as JR  # noqa: E402
import ycc_restate as Y  # noqa: E402

EXTRA = [(31, 31), (32, 32), (33, 33), (31, 33), (33, 32), (171, 129), (341, 255), (455, 256), (336, 256)]
CONTROL = (340, 256)  # the usual flow size (a partial block column); 336 x 256 and 32 x 32 are whole MCUs
GRAY_SIZES = [(w, h) for w in range(1, 18) for h in range(1, 18)] + EXTRA + [CONTROL]
COLOUR_SIZES = GRAY_SIZES + [(107, 80), (1920, 1080), (2047, 1151)]
MAXW, MAXH = 2048, 1152

_handles = []


def handle(w=MAXW, h=MAXH, alg="tvl1"):
    import denseflow_b200 as d
    e = d.create(alg, 0, w, h).set("jpeg_exact", 0)
    _handles.append(e)
    return e


@pytest.fixture(autouse=True)
def _release():
    """every handle a test made is destroyed when the test ends, so device memory does not pile up over the module"""
    yield
    for e in _handles:
        e.release()
    _handles.clear()


def r8(x):
    return -(-x // 8) * 8


def r16(x):
    return -(-x // 16) * 16


def resized(w, h):
    """a destination size for the resize arms: another partial-block size near (w, h)"""
    return (max(1, w + 3 - 2 * (w % 3)), max(1, h - 1 + 2 * (h % 2)))


def noise(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def colour_frames(n, w, h, seed=0, shift=1):
    """n smooth colour frames with texture, each shifted `shift` px right of the last (motion for the flow chains)"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (max(h // 4, 1) + 3, max(w // 4, 1) + 3 + n * shift, 3), dtype=np.uint8)
    big = cv2.resize(base, (base.shape[1] * 4, base.shape[0] * 4), interpolation=cv2.INTER_CUBIC)
    big = np.clip(big.astype(np.int16) + rng.integers(-6, 7, big.shape), 0, 255).astype(np.uint8)
    return [np.ascontiguousarray(big[:h, k * shift:k * shift + w]) for k in range(n)]


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED)


# ---- a. bytes are a function of the image ------------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", GRAY_SIZES)
def test_gray_device_bytes_ignore_memory_around_the_plane(w, h):
    import torch
    e = handle(512, 288)
    img = noise((h, w), w * 100 + h) if (w + h) % 2 else np.asarray(cv2.resize(noise((4, 4), w + h), (w, h), interpolation=cv2.INTER_CUBIC))
    files = []
    for k, extra in enumerate((1 + (w * 7 + h) % 67, 67, 1)):
        for poison in ("zero", "ones", "noise"):
            pitch = w + extra
            rows = h + 16 + (w % 5)
            buf = {"zero": np.zeros((rows, pitch), np.uint8), "ones": np.full((rows, pitch), 255, np.uint8),
                   "noise": noise((rows, pitch), 7 + k)}[poison]
            buf[:h, :w] = img
            dev = torch.from_numpy(buf).cuda()
            files.append(e.encode_jpeg_gray_device(dev[:h, :w], 95))
    assert all(f == files[0] for f in files), [len(f) for f in files]
    assert imdecode(files[0]).shape == (h, w)


def _dirty_gray(e):
    """fills the flow chain's scratch with the planes of a larger noise call"""
    frames = [noise((256, 455, 3), s) for s in range(19)]
    e.process_bgr_batch(frames, 1)


def _dirty_colour(e):
    """fills the frame-extraction scratch with the planes of a larger noise call"""
    e.extract_frames([noise((1151, 2047, 3), s) for s in range(17)])


CHAIN_CASES = [((9, 7), 2, 1), ((17, 13), 9, -1), ((31, 33), 19, 3), ((13, 17), 10, 1), ((107, 80), 11, -1),
               ((171, 129), 12, 3), ((341, 255), 9, 1), ((33, 32), 5, 3), ((3, 5), 4, 1), (CONTROL, 4, 1)]


@pytest.mark.parametrize("resize", [False, True])
@pytest.mark.parametrize("source", ["bgr", "jpeg"])
def test_flow_chain_bytes_ignore_scratch_history(source, resize):
    clean, dirty = handle(512, 288), handle(512, 288)
    _dirty_gray(dirty)
    for (w, h), n, step in CHAIN_CASES:
        frames = colour_frames(n, w, h, seed=w + h, shift=1)
        new_size = resized(w, h) if resize and (w, h) != CONTROL else None
        if source == "bgr":
            run = lambda e: e.process_bgr_batch(frames, step, 20, new_size)  # noqa: E731
        else:
            files = [cv2.imencode(".jpg", f)[1].tobytes() for f in frames]
            run = lambda e: e.process_jpeg_batch(files, step, 20, new_size)  # noqa: E731
        a, b = run(clean), run(dirty)
        assert len(a) == n - abs(step)
        assert a == b, ((w, h), n, step, new_size)


@pytest.mark.parametrize("resize", [False, True])
@pytest.mark.parametrize("source", ["bgr", "jpeg"])
def test_extract_bytes_ignore_scratch_history(source, resize):
    clean, dirty = handle(), handle()
    _dirty_colour(dirty)
    cases = [((w, h), n) for (w, h), n in zip([(1, 1), (7, 9), (17, 16), (15, 17), (33, 31), (107, 80), (171, 129),
                                                 (1920, 1080), (2047, 1151), CONTROL], [1, 8, 9, 17, 9, 8, 17, 9, 17, 8])]
    for (w, h), n in cases:
        frames = colour_frames(n, w, h, seed=w * h)
        new_size = resized(w, h) if resize and (w, h) != CONTROL else None
        if source == "bgr":
            run = lambda e: e.extract_frames(frames, new_size)  # noqa: E731
        else:
            files = [cv2.imencode(".jpg", f)[1].tobytes() for f in frames]
            run = lambda e: e.extract_frames_jpeg(files, new_size)  # noqa: E731
        a, b = run(clean), run(dirty)
        assert a == b, ((w, h), n, new_size)


@pytest.mark.parametrize("resize", [False, True])
def test_bgr_device_bytes_ignore_scratch_history(resize):
    import torch
    clean, dirty = handle(), handle()
    _dirty_colour(dirty)
    dirty.encode_jpeg_bgr_device(torch.from_numpy(noise((1151, 2047, 3), 3)).cuda())
    got = {}
    for order, e in ((COLOUR_SIZES, clean), (COLOUR_SIZES[::-1], dirty)):  # each handle sees the sizes in another order
        for w, h in order:
            img = torch.from_numpy(colour_frames(1, w, h, seed=w + 3 * h)[0]).cuda()
            new_size = resized(w, h) if resize and (w, h) != CONTROL else None
            got.setdefault((w, h), []).append(e.encode_jpeg_bgr_device(img, new_size))
    for k, (a, b) in got.items():
        assert a == b, k


def test_run_videos_files_ignore_worker_history():
    """two workers on one device; noise videos larger than the partial-MCU ones between them, in two orders"""
    from denseflow_b200 import listrun
    small = [colour_frames(n, w, h, seed=w + h) for (w, h), n in [((107, 80), 9), ((33, 17), 7), ((171, 129), 10), ((15, 9), 6)]]
    big = [[noise((256, 455, 3), 10 * v + s) for s in range(8)] for v in range(3)]
    videos = [small[0], big[0], small[1], big[1], small[2], big[2], small[3]]
    r = listrun.ListRunner("tvl1", [0, 0], 512, 288)
    try:
        _check_list_runs(r, videos)
    finally:
        r.close()


def _check_list_runs(r, videos):
    def run(order, step):
        got = {i: {} for i in order}
        lock = threading.Lock()
        per = 2 if step else 1

        def on_chunk(video, dev, first, last, files):
            with lock:
                for k, f in enumerate(files):
                    got[order[video]][per * first + k] = bytes(f)

        r.run_videos([videos[i] for i in order], step=step, chunk_flows=4, on_chunk=on_chunk)
        return {i: [got[i][k] for k in range(len(got[i]))] for i in order}

    for step in (0, 1):
        fwd = run(list(range(len(videos))), step)
        rev = run(list(range(len(videos)))[::-1], step)
        for i in (0, 2, 4, 6):
            e = handle(512, 288)
            if step == 0:
                want = e.extract_frames(videos[i])
            else:
                want = [f for p in e.process_bgr_batch(videos[i], step) for f in p]
            assert fwd[i] == want and rev[i] == want, (i, step)


# ---- b. the padded planes are libjpeg's ---------------------------------------------------------------------------------

def padded_ycc_want(bgr, dw, dh):
    """Y edge-replicated to whole MCUs, Cb / Cr as jpeg_encode_restate.chroma_padded pads them"""
    img = Y.resize_linear_u8c(bgr, dw, dh) if (dw, dh) != bgr.shape[1::-1] else bgr
    yy, cb, cr = Y.bgr_to_ycc(img)
    return (JR._pad_edge(yy.astype(np.uint8), r16(dh), r16(dw)), JR.chroma_padded(cb, dw, dh), JR.chroma_padded(cr, dw, dh))


@pytest.mark.parametrize("resize", [False, True])
def test_padded_ycc_planes_are_libjpegs(resize):
    e = handle()
    for w, h in COLOUR_SIZES:
        bgr = noise((h, w, 3), w * 7 + h)
        dw, dh = resized(w, h) if resize and (w, h) != CONTROL else (w, h)
        cw, ch = r8((dw + 1) // 2), r8((dh + 1) // 2)
        outs, _ = e.debug_run_kernel("jpeg_padded_ycc420", [bgr[..., c] for c in range(3)], 3, scalars=(dw, dh),
                                     out_shape=[(2 * ch, 2 * cw), (ch, cw), (ch, cw)])
        want = padded_ycc_want(bgr, dw, dh)
        for name, got, ref in zip("Y Cb Cr".split(), outs, want):
            assert got.shape == ref.shape and np.array_equal(got, ref), (name, (w, h), (dw, dh))


def test_padded_gray_planes_are_libjpegs():
    import torch
    e = handle(512, 288)
    for w, h in GRAY_SIZES:
        img = noise((h, w), w * 31 + h)
        (got,), _ = e.debug_run_kernel("jpeg_padded_gray", [img], 1, out_shape=(r8(h), r8(w)))
        want = JR._pad_edge(img, r8(h), r8(w))
        assert np.array_equal(got, want), (w, h)
        # the file is nvJPEG's of that padded plane, handed over from a buffer of exactly the padded size
        exact = torch.from_numpy(np.ascontiguousarray(want)).cuda()
        loose = torch.from_numpy(np.pad(img, ((0, 9), (0, 13)), constant_values=0x5A)).cuda()
        assert e.encode_jpeg_gray_device(exact[:h, :w]) == e.encode_jpeg_gray_device(loose[:h, :w]), (w, h)


# ---- c. edge quality against imencode -------------------------------------------------------------------------------------

# Margins over imencode's error, from the residuals measured on an H100 80GB HBM3 at a 700 W power limit: a block may exceed
# imencode's whole-image maximum by BLOCK_MARGIN, the last block row or column imencode's maximum on that band by BAND_MARGIN.
GRAY_MARGINS = (4, 4)      # measured: 3 and 3 (6 x 13 noise)
COLOUR_MARGINS = (10, 10)  # measured: 8 and 8 (5 x 12 resized to 4 x 11); nvJPEG gave the same before its planes were padded


def edge_errors(dec, ref_dec, img):
    """(worst block excess over imencode's image max, worst band excess over imencode's band max), both int"""
    h, w = img.shape[:2]
    err = np.abs(dec.astype(int) - img.astype(int))
    rerr = np.abs(ref_dec.astype(int) - img.astype(int))
    if err.ndim == 3:
        err, rerr = err.max(2), rerr.max(2)
    block = max(int(err[y:y + 8, x:x + 8].max()) for y in range(0, h, 8) for x in range(0, w, 8)) - int(rerr.max())
    by, bx = (h - 1) // 8 * 8, (w - 1) // 8 * 8
    band = max(int(err[by:].max()) - int(rerr[by:].max()), int(err[:, bx:].max()) - int(rerr[:, bx:].max()))
    return block, band


def check_edges(cases, margins, what):
    """cases: (label, decoded nvJPEG file, decoded imencode file, image); every case within margins, worst printed"""
    res = [(label,) + edge_errors(dec, ref_dec, img) for label, dec, ref_dec, img in cases]
    worst_block, worst_band = max(res, key=lambda r: r[1]), max(res, key=lambda r: r[2])
    print("%s: worst block excess %d at %s, worst edge band excess %d at %s" % (what, worst_block[1], worst_block[0], worst_band[2],
                                                                                worst_band[0]))
    bad = [r for r in res if r[1] > margins[0] or r[2] > margins[1]]
    assert not bad, bad[:10]


def test_gray_edges_decode_like_imencode(oracle):
    import torch
    e = handle(512, 288)
    planes = []
    for w, h in [(17, 13), (33, 31), (171, 129), (341, 255), CONTROL]:
        a, b, _ = synth.pair(h, w, w)
        planes += list(oracle.quantise(oracle.tvl1_calc(a, b), 20))
    planes += [noise((h, w), w + 17 * h) for w, h in GRAY_SIZES]
    cases = []
    for img in planes:
        dec = imdecode(e.encode_jpeg_gray_device(torch.from_numpy(np.ascontiguousarray(img)).cuda(), 95))
        cases.append((img.shape[::-1], dec, imdecode(cv2.imencode(".jpg", img)[1]), img))
    check_edges(cases, GRAY_MARGINS, "gray")


@pytest.mark.parametrize("resize", [False, True])
def test_colour_edges_decode_like_imencode(resize):
    import torch
    e = handle()
    cases = []
    for w, h in COLOUR_SIZES:
        bgr = colour_frames(1, w, h, seed=5 * w + h)[0]
        new_size = resized(w, h) if resize and (w, h) != CONTROL else None
        img = Y.resize_linear_u8c(bgr, *new_size) if new_size else bgr
        dec = cv2.imdecode(np.frombuffer(e.encode_jpeg_bgr_device(torch.from_numpy(bgr).cuda(), new_size), np.uint8), cv2.IMREAD_COLOR)
        cases.append(((w, h, new_size), dec, cv2.imdecode(cv2.imencode(".jpg", img)[1], cv2.IMREAD_COLOR), img))
    check_edges(cases, COLOUR_MARGINS, "colour")
