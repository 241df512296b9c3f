"""The PNG restatement (tests/png_restate.py) pinned to cv2.imencode(".png") and to golden bytes, and the zlib rules the GPU
encoder (denseflow_b200/csrc/png_encode.cu) restates, read back from the restatement's streams with tests/inflate_trace.py."""
import os

import numpy as np
import pytest

import inflate_trace as T
import png_cases as PC
import png_restate as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png_imencode_cases.npz")


def _stream(img):
    return P.zlib_stream(P.scanlines(img))


@pytest.mark.parametrize("kind", PC.CONTENTS)
def test_restatement_equals_imencode(kind):
    cv2 = pytest.importorskip("cv2")
    for h, w in PC.PROBE_SIZES:
        img = PC.image(kind, h, w)
        ok, want = cv2.imencode(".png", img)
        assert ok
        got = P.encode(img)
        assert got == want.tobytes(), ((h, w), T.first_difference(P.idat_stream(got), P.idat_stream(want.tobytes())))


@pytest.mark.parametrize("n", [3, 4, 5, 257, 258, 259, 260, 261, 262, 516, 517, 518, 519])
def test_runs_of_exact_lengths(n):
    cv2 = pytest.importorskip("cv2")
    img = PC.run_image(n)
    raw = P.scanlines(img)
    assert bytes(n) in raw and bytes(n + 1) not in raw
    blocks, data = T.trace(_stream(img))
    assert data == raw
    assert [s for b in blocks for s in b["symbols"]] == PC.rle_parse(raw)
    assert P.encode(img) == cv2.imencode(".png", img)[1].tobytes()


@pytest.mark.parametrize("shape", [(3, 100), (40, 87), (7, 1), (1, 7)])
def test_runs_across_scanlines(shape):
    """Filter bytes are part of the stream: a run of ones spans every scanline of the ramp."""
    cv2 = pytest.importorskip("cv2")
    img = PC.ramp(*shape)
    raw = P.scanlines(img)
    blocks, _ = T.trace(_stream(img))
    syms = [s for b in blocks for s in b["symbols"]]
    assert syms == PC.rle_parse(raw)
    if shape[1] > 1:
        assert set(raw) == {1}
        assert sum(s[0] for s in syms if isinstance(s, tuple)) == len(raw) - 1
    assert P.encode(img) == cv2.imencode(".png", img)[1].tobytes()


@pytest.mark.parametrize("shape", PC.BLOCK_EDGE_SIZES)
def test_block_split_on_literal_noise(shape):
    """16383 symbols per block; when the last block is full, an empty final block follows"""
    cv2 = pytest.importorskip("cv2")
    h, w = shape
    img = PC.literal_noise(h, w)
    raw = P.scanlines(img)
    assert len(raw) % 16383 == 0
    blocks, _ = T.trace(_stream(img))
    k = len(raw) // 16383
    assert [b["type"] for b in blocks] == ["stored"] * k + ["fixed"]
    assert [b.get("stored_len") for b in blocks[:k]] == [16383] * k
    assert blocks[-1]["symbols"] == [] and blocks[-1]["final"] == 1
    assert P.encode(img) == cv2.imencode(".png", img)[1].tobytes()
    # one more byte per row: the last block holds the leftover symbols, no empty block
    img2 = PC.literal_noise(h + 1, w)
    blocks2, _ = T.trace(_stream(img2))
    assert [b["type"] for b in blocks2][:k] == ["stored"] * k and len(blocks2) == k + 1
    assert blocks2[-1]["final"] == 1 and blocks2[-1].get("stored_len") == len(P.scanlines(img2)) - 16383 * k


def test_block_kinds():
    noise = T.trace(_stream(PC.image("noise", 64, 200)))[0]
    assert {b["type"] for b in noise} == {"stored"}
    smooth = T.trace(_stream(PC.image("smooth", 256, 340)))[0]
    assert {b["type"] for b in smooth} == {"dynamic"}
    assert all(len(b["symbols"]) == 16383 for b in smooth[:-1])
    tiny = T.trace(_stream(PC.image("constant", 2, 2)))[0]
    assert [b["type"] for b in tiny] == ["fixed"]


def test_stored_blocks_stay_inside_the_window():
    """zlib offers a stored block only while its bytes are still in the 32 KB window; stored blocks never come close to the
    32 506 bytes where that would bind, so the encoder need not model the window."""
    for kind, h, w in [("mixed", 256, 340), ("noise", 256, 340), ("mixed", 90, 91)]:
        for b in T.trace(_stream(PC.image(kind, h, w)))[0]:
            if b["type"] == "stored":
                assert b["stored_len"] <= 16383 + 2 * 258


def test_golden_bytes():
    cv2 = pytest.importorskip("cv2")
    g = np.load(GOLDEN)
    n = sum(1 for k in g.files if k.startswith("img"))
    assert n >= 5
    for i in range(n):
        img, want = g["img%d" % i], g["png%d" % i].tobytes()
        assert P.encode(img) == want, (i, T.first_difference(P.idat_stream(P.encode(img)), P.idat_stream(want)))
        assert np.array_equal(cv2.imdecode(np.frombuffer(want, np.uint8), cv2.IMREAD_COLOR), img)


def test_max_bytes_bounds_the_file():
    from denseflow_b200 import _lib
    L = _lib.load("default")
    assert L.dfb_png_max_bytes(0, 5) == 0 and L.dfb_png_max_bytes(5, -1) == 0
    for h, w in PC.PROBE_SIZES + PC.BLOCK_EDGE_SIZES:
        assert L.dfb_png_max_bytes(w, h) >= len(P.encode(PC.image("noise", h, w))), (h, w)
    for h, w in PC.BLOCK_EDGE_SIZES:
        assert L.dfb_png_max_bytes(w, h) >= len(P.encode(PC.literal_noise(h, w)))
