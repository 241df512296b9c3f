"""The restatement of cv2.imdecode (tests/jpeg_restate.py) pinned live to cv2 and to the golden fixture: byte-equal BGR and
gray over every small size, sampling, quality and the encoder options a frame folder can hold, plus the refusals."""
import os

import cv2
import numpy as np
import pytest

import jpeg_cases as J
import jpeg_restate as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_decode_cases.npz")


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def check(b):
    want = imdecode(b)
    got = R.decode(b)
    assert got.shape == want.shape and np.array_equal(got, want)
    assert np.array_equal(R.bgr_to_gray(got), cv2.cvtColor(want, cv2.COLOR_BGR2GRAY))


@pytest.mark.parametrize("sampling", J.SAMPLINGS)
@pytest.mark.parametrize("quality", [1, 50, 95, 100])
@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_every_small_size(sampling, quality, kind):
    # 1..17 covers chroma planes of 1, 2 and 3+ samples (box vs triangle upsampling) and partial MCUs on both axes
    for h in range(1, 18):
        for w in range(1, 18):
            check(J.encode(J.image(kind, h, w), sampling, quality))


@pytest.mark.parametrize("sampling", J.SAMPLINGS)
@pytest.mark.parametrize("restart", [1, 2, 7])
def test_restart_intervals(sampling, restart):
    check(J.encode(J.image("noise", 45, 61), sampling, 95, restart=restart))
    check(J.encode(J.image("smooth", 33, 70), sampling, 75, restart=restart))


@pytest.mark.parametrize("sampling", J.SAMPLINGS)
def test_optimized_huffman_tables_and_split_qualities(sampling):
    check(J.encode(J.image("smooth", 45, 61), sampling, 95, optimize=True))
    check(J.encode(J.image("noise", 45, 61), sampling, 100, optimize=True))
    check(J.encode(J.image("noise", 45, 61), sampling, 95, luma=90, chroma=30))


@pytest.mark.parametrize("h,w", [(256, 340), (720, 1280)])
def test_frame_sizes(h, w):
    check(J.encode(J.image("smooth", h, w), "420", 95))


def test_pillow_files():
    files = J.pillow_files()
    b = files["qt16"]
    i = b.index(b"\xff\xdb")
    assert b[i + 4] >> 4 == 1  # the first DQT table has 16-bit values
    assert b"frame folder" in files["exif1_com"] and b"Exif" in files["exif1_com"]
    for b in files.values():
        check(b)


@pytest.mark.parametrize("name", sorted(J.refusals()))
def test_refusals(name):
    b, kind, frag = J.refusals()[name]
    with pytest.raises(R.Unsupported if kind == "unsupported" else R.Corrupt, match=frag):
        R.decode(b)
    if name != "orientation6":
        assert imdecode(b) is not None  # libjpeg decodes these (with warnings); the restatement refuses


def test_golden_fixture():
    g = np.load(GOLDEN)
    n = int(g["n"])
    assert n >= 8
    for i in range(n):
        b = g["jpg%d" % i].tobytes()
        assert np.array_equal(R.decode(b), g["bgr%d" % i])
        assert np.array_equal(imdecode(b), g["bgr%d" % i])
