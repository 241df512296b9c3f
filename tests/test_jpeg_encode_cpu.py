"""The numpy restatement of libjpeg-turbo's compressor (tests/jpeg_encode_restate.py) against cv2.imencode(".jpg") live,
byte for byte: small sizes at every block and MCU edge, five qualities, several kinds of content, real quantised flow planes,
two large sizes, the entropy coder's edge cases, and the committed fixture the GPU tests also read."""
import os

import numpy as np
import pytest

import jpeg_encode_cases as JC
import jpeg_encode_restate as E
import ycc_restate as Y

cv2 = pytest.importorskip("cv2")

SMALL = list(range(1, 18)) + [31, 32, 33]
QUALITIES = (1, 50, 75, 95, 100)
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_encode_cases.npz")


def imencode(img, q=95):
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, int(q)])[1].tobytes()


def _same(got, want, what=""):
    assert got == want, (what, E.locate(got, want))


def _content(kind, h, w, colour, seed):
    rng = np.random.default_rng(seed)
    shape = (h, w, 3) if colour else (h, w)
    if kind == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "constant":
        return np.full(shape, 201, np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    s = (128 + 100 * np.sin(xx / 5.0) * np.cos(yy / 7.0)).astype(np.uint8)
    return np.stack([s, 255 - s, np.roll(s, 3, 1)], -1) if colour else s


@pytest.mark.parametrize("colour", [False, True])
@pytest.mark.parametrize("kind", ["noise", "constant", "smooth"])
def test_small_sizes(kind, colour):
    for q in QUALITIES:
        for h in SMALL:
            for w in SMALL:
                img = _content(kind, h, w, colour, 1000 * h + w)
                _same(E.encode(img, q), imencode(img, q), (kind, colour, w, h, q))


@pytest.mark.parametrize("w, h", [(340, 256), (1280, 720)])
def test_large_sizes(w, h):
    rng = np.random.default_rng(w)
    smooth = cv2.resize(rng.integers(0, 256, (h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8), (w, h))
    img = (smooth.astype(np.int16) + rng.integers(-12, 13, smooth.shape)).clip(0, 255).astype(np.uint8)
    _same(E.encode(img, 95), imencode(img, 95), "bgr")
    _same(E.encode(img[..., 0], 95), imencode(np.ascontiguousarray(img[..., 0]), 95), "gray")


def test_quantised_flow_planes(oracle):
    """real flow planes: synth.pair through the TV-L1 oracle and oracle.quantise, as `-st=jpg` writes them"""
    from denseflow_b200 import synth
    f0, f1, _ = synth.pair(64, 96, seed=4)
    flow = oracle.tvl1_calc(f0, f1)
    for bound in (5, 20):
        for q in (75, 95):
            for plane in oracle.quantise(flow, bound):
                _same(E.encode(plane, q), imencode(plane, q), (bound, q))


def test_entropy_edge_cases_hit_their_edges():
    """each constructed case really produces the coefficient pattern it is named for"""
    for name, img, q, z in JC.run_cases():
        zz = JC.zz_coefficients(img, q)
        nz = np.flatnonzero(zz[0, 1:]) + 1
        assert list(nz) == [z], (name, list(nz))
    coef, _ = E.coefficients(JC.dc_category11(), 100)
    diffs = np.diff(coef[:, 0])
    assert int(np.abs(diffs).max()).bit_length() == 11
    data = E.entropy(*E.coefficients(JC.ff_flush_case(), 50))
    assert data.endswith(b"\xff\x00")


def test_entropy_edge_cases_against_cv2():
    for name, img, q in JC.entropy_cases():
        want = imencode(img, q)
        _same(E.encode(img, q), want, name)
        if name.startswith("ff_"):
            assert b"\xff\x00" in want, name


def test_chroma_bottom_padding_rule():
    """the rule the byte pin confirms: chroma rows past ceil(h / 2) replicate the last downsampled row.  At an even height
    the replication of full-resolution rows up to the MCU (ycc_restate.mcu_padded) gives other padding samples, so the pin
    tells the two apart (at an odd height they coincide)"""
    img = np.random.default_rng(21).integers(0, 256, (18, 21, 3), dtype=np.uint8)
    want = imencode(img)
    _same(E.encode(img), want)
    h, w = img.shape[:2]
    _, cb, _ = Y.bgr_to_ycc(Y.mcu_padded(img))
    full_rows = E.chroma_padded(cb[:, :w], w, 2 * ((h + 15) // 16) * 8)
    _, cb0, _ = Y.bgr_to_ycc(img)
    assert not np.array_equal(full_rows, E.chroma_padded(cb0, w, h))


def test_golden_fixture_matches_cv2():
    z = np.load(GOLDEN)
    names = [k[4:] for k in z.files if k.startswith("img_")]
    assert len(names) >= 10
    for n in names:
        img, q, want = z["img_" + n], int(z["q_" + n]), z["jpg_" + n].tobytes()
        _same(imencode(img, q), want, n)
        _same(E.encode(img, q), want, n)
