"""The frame-extraction restatement (tests/ycc_restate.py) against the real code imencode(".jpg") runs: cv2.resize on
CV_8UC3, and libjpeg-turbo's colour conversion and 4:2:0 downsampling (through cv2.imencode, read back with Pillow).

Pillow's draft("YCbCr", ...) turns off libjpeg's output colour conversion; at half scale libjpeg decodes the chroma
components with a full 8 x 8 IDCT, so the planes come back at their native resolution.  At quality 100 every quantiser
step is 1, and a block whose samples are all equal holds a DC coefficient only, which decodes back exactly: the images
below are built from such blocks, so the decoded samples are the encoder's own input samples."""
import io

import numpy as np
import pytest

import geometry_cases as gc
import ycc_restate as Y

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")


def _encode_q100(bgr):
    ok, buf = cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 100])
    assert ok
    return buf.tobytes()


def _decode_ycc(jpg, half):
    """the decoded Y, Cb, Cr planes without colour conversion; half: decode at scale 1/2 (chroma at native resolution)"""
    im = Image.open(io.BytesIO(jpg))
    w, h = im.size
    im.draft("YCbCr", (w // 2, h // 2) if half else (w, h))
    assert im.mode == "YCbCr" and im.size == (((w + 1) // 2, (h + 1) // 2) if half else (w, h))
    a = np.asarray(im)
    return a[..., 0], a[..., 1], a[..., 2]


@pytest.mark.parametrize("src, dst", [((1920, 1080), (340, 256)), ((1920, 1080), (960, 540)), ((320, 240), (640, 480)),
                                      ((37, 23), (5, 3)), ((641, 479), (1, 1)), ((100, 3), (7, 201)), ((1920, 1080), (455, 256)),
                                      ((320, 240), (320, 240))])
def test_colour_resize_matches_opencv(src, dst):
    (sw, sh), (dw, dh) = src, dst
    bgr = np.random.default_rng(sw + 3 * dh).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    assert np.array_equal(Y.resize_linear_u8c(bgr, dw, dh), cv2.resize(bgr, (dw, dh)))


@pytest.mark.parametrize("src, dst", gc.RESIZE_CASES)
def test_colour_resize_matches_opencv_at_degenerate_sizes(src, dst):
    (sw, sh), (dw, dh) = src, dst
    bgr = np.random.default_rng(sw * 7 + sh).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    assert np.array_equal(Y.resize_linear_u8c(bgr, dw, dh), cv2.resize(bgr, (dw, dh), interpolation=cv2.INTER_LINEAR))


def test_colour_conversion_matches_libjpeg():
    """16 384 random colours, one per constant 16 x 16 MCU: the decoded Y, Cb, Cr at every MCU centre are rgb_ycc_convert's"""
    rng = np.random.default_rng(5)
    n = 128
    cols = rng.integers(0, 256, (n, n, 3), dtype=np.uint8)
    bgr = np.repeat(np.repeat(cols, 16, 0), 16, 1)
    y, cb, cr = _decode_ycc(_encode_q100(bgr), half=False)
    want = Y.bgr_to_ycc(cols)
    for got, ref in zip((y, cb, cr), want):
        assert np.array_equal(got[8::16, 8::16].astype(np.int64), ref)


def _pattern_image(rng, mh, mw):
    """mh x mw MCUs, each tiled with one random 2 x 2 BGR pattern"""
    pat = rng.integers(0, 256, (mh, mw, 2, 2, 3), dtype=np.uint8)
    return np.tile(pat, (1, 1, 8, 8, 1)).transpose(0, 2, 1, 3, 4).reshape(mh * 16, mw * 16, 3)


def test_downsampling_bias_matches_libjpeg():
    """3 072 MCUs tiled with a random 2 x 2 pattern each: the decoded chroma equals h2v2_downsample's alternating 1 / 2 bias
    inside every 8 x 8 chroma block (221 184 samples), and a constant bias of 2 does not"""
    rng = np.random.default_rng(11)
    bgr = _pattern_image(rng, 48, 64)
    _, cb, cr = _decode_ycc(_encode_q100(bgr), half=True)
    _, rcb, rcr = Y.bgr_to_ycc420(bgr)
    edge = lambda n: np.arange(n) % 8 % 7 == 0  # first and last sample of every 8 x 8 chroma block
    inner = ~edge(cb.shape[0])[:, None] & ~edge(cb.shape[1])[None, :]
    assert inner.sum() * 2 == 221184
    for got, ref in ((cb, rcb), (cr, rcr)):
        assert np.array_equal(got[inner], ref[inner])
    # the model with one constant bias is told apart
    _, ycb, ycr = Y.bgr_to_ycc(bgr)
    const = lambda c: ((c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    wrong = int((const(ycb)[inner] != cb[inner]).sum() + (const(ycr)[inner] != cr[inner]).sum())
    print("constant-bias model mismatches:", wrong)
    assert wrong > 1000


def _chroma(bgr):
    cb, cr = Y.bgr_to_ycc(bgr[None, None])[1:]
    return int(cb[0, 0]), int(cr[0, 0])


def _edge_image(rng, w, h):
    """A w x h frame whose every chroma block, after libjpeg's edge replication, holds one value (so q100 decodes it
    exactly): each MCU has even rows of colour A and odd rows of colour B with Cb_A + Cb_B and Cr_A + Cr_B even; in the
    bottom MCU row, B is A shifted along the gray axis (same Cb and Cr), as the replicated last row then fills the block."""
    img = np.empty((h, w, 3), np.uint8)
    for y0 in range(0, h, 16):
        for x0 in range(0, w, 16):
            while True:
                a = rng.integers(16, 240, 3)
                if y0 + 16 >= h:
                    b = np.clip(a + rng.integers(-16, 17), 0, 255)
                    if _chroma(b.astype(np.uint8)) == _chroma(a.astype(np.uint8)):
                        break
                else:
                    b = rng.integers(0, 256, 3)
                    ca, cb_ = _chroma(a.astype(np.uint8)), _chroma(b.astype(np.uint8))
                    if (ca[0] + cb_[0]) % 2 == 0 and (ca[1] + cb_[1]) % 2 == 0:
                        break
            blk = img[y0:y0 + 16, x0:x0 + 16]
            blk[0::2] = a
            blk[1::2] = b
    return img


@pytest.mark.parametrize("w, h", [(17, 16), (16, 17), (17, 17), (31, 33), (47, 45), (15, 15), (1, 1), (1, 2), (2, 1), (1, 37), (37, 1),
                                  (3, 1), (1, 3), (33, 2), (99, 67)])
def test_odd_edges_replicate_like_libjpeg(w, h):
    """odd widths and heights, 1 x 1, 1 x N, N x 1: the decoded chroma equals the restatement's, whose last column / row
    pairs with itself; pairing the missing sample with zero instead is told apart wherever the frame has an odd edge"""
    rng = np.random.default_rng(w * 131 + h)
    bgr = _edge_image(rng, w, h)
    _, rcb, rcr = Y.bgr_to_ycc420(bgr)
    ch, cw = rcb.shape
    assert (ch, cw) == ((h + 1) // 2, (w + 1) // 2)
    if w >= 2 and h >= 2:
        _, cb, cr = _decode_ycc(_encode_q100(bgr), half=True)
        mask = np.ones((ch, cw), bool)
    else:
        # a one-pixel side cannot be halved: decode at full scale, where libjpeg's fancy upsampler mixes each chroma sample
        # with its neighbours (the edge sample with itself); where all of them lie in the same block it returns the sample
        _, cb, cr = (p[0::2, 0::2] for p in _decode_ycc(_encode_q100(bgr), half=False))
        same = lambda n: (np.clip(np.arange(n) - 1, 0, n - 1) // 8 == np.arange(n) // 8) & \
                         (np.clip(np.arange(n) + 1, 0, n - 1) // 8 == np.arange(n) // 8)
        mask = same(ch)[:, None] & same(cw)[None, :]
        assert mask[-1, -1]
    assert cb.shape == rcb.shape
    assert np.array_equal(cb[mask], rcb[mask]) and np.array_equal(cr[mask], rcr[mask])
    # the padded frame's chroma is constant per 8 x 8 block: the precondition of the exact decode
    _, pcb, pcr = Y.bgr_to_ycc420(Y.mcu_padded(bgr))
    for p in (pcb, pcr):
        blocks = p.reshape(p.shape[0] // 8, 8, p.shape[1] // 8, 8)
        assert (blocks == blocks[:, :1, :, :1]).all()
    if w % 2 or h % 2:
        _, ycb, _ = Y.bgr_to_ycc(bgr)
        z = np.pad(ycb, ((0, h & 1), (0, w & 1)))  # a missing sample taken as zero
        s = z[0::2, 0::2] + z[0::2, 1::2] + z[1::2, 0::2] + z[1::2, 1::2]
        zero = ((s + 1 + (np.arange(s.shape[1]) & 1)) >> 2).astype(np.uint8)
        assert not np.array_equal(zero[mask], cb[mask])
