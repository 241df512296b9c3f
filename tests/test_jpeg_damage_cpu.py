"""Damaged and hand-built JPEG files (tests/jpeg_damage_cases.py) against cv2.imdecode and the decoder's header parser:
every file the restatement accepts decodes to imdecode's bytes, every file imdecode refuses the restatement refuses too,
dfb_jpeg_info gives the restatement's header verdict, and the out-of-range bound is derived from the encoder."""
import collections

import cv2
import numpy as np
import pytest

import jpeg_damage_cases as D
import jpeg_encode_restate as E
import jpeg_restate as R


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


_CASES = D.all_cases()


def test_the_cases_reach_their_edges():
    by = collections.defaultdict(collections.Counter)
    for name, (b, edge) in _CASES.items():
        by[edge][D.verdict(b)] += 1
    kinds = {v for c in by.values() for v in c}
    for k in ("code", "short", "rst", "rst_count", "range", "no_end"):
        assert ("corrupt", k) in kinds, k
    assert ("ok", None) in by["bitflip"] and ("ok", None) in by["dequant"]
    for edge in ("bitflip", "truncate", "marker", "rst", "junk", "fill", "no_eoi", "order", "run63", "eob63", "dc_wrap"):
        assert by[edge], edge
    # an interval that ends early before one holding an invalid code: the invalid code is the file's error, as is one before
    assert D.verdict(_CASES["gray_ri3/short_then_code"][0]) == ("corrupt", "code")
    assert D.verdict(_CASES["gray_ri3/code_then_short"][0]) == ("corrupt", "code")
    # every header refusal of the decoder's parser is reached by a named case
    msgs = {D.verdict(b) for b in D.header_cases().values()}
    for m in ["bad Huffman table", "bad DHT table id", "short DHT segment", "bad DQT table id", "short DQT segment",
              "short frame header", "short scan header", "short DRI segment", "scan uses an undefined table",
              "scan component does not match the frame", "bad spectral selection in a sequential scan",
              "marker segment runs past the end of the file", "garbage between markers", "not a JPEG file (no SOI marker)",
              "file ends before the scan", "scan before the frame header", "unexpected marker before the scan"]:
        assert ("corrupt", m) in msgs, m


def test_hand_built_files_decode_to_what_was_written():
    # the writer: coefficient blocks in, the restatement's coefficients out
    blk = np.zeros((4 * 6, 64), np.int64)  # 32 x 32 4:2:0: 2 x 2 MCUs of 6 blocks
    rng = np.random.default_rng(1)
    blk[:, :10] = rng.integers(-60, 60, (24, 10))
    blk[:, 0] = rng.integers(-900, 900, 24)
    for ri in (0, 1, 3):
        b = D.write(32, 32, "420", blk, ri=ri)
        assert np.array_equal(R.coefficients(R.parse(b)), blk)
    got = R.coefficients(R.parse(D.coefficient_cases()["zrl_past_63"][0]))
    assert got[0, 0] == 10 and got[0, 1] == 3 and (got[0, 2:] == 0).all()  # ZRLs past index 63 end the block
    got = R.coefficients(R.parse(D.coefficient_cases()["run_past_63"][0]))
    assert got[0, 63] == -7 and (got[0, 1:63] == 0).all()  # 1 + 3 x 16 + a run of 15 places the value at 63, as libjpeg
    got = R.coefficients(R.parse(D.coefficient_cases()["dc_wrap_up"][0]))
    assert list(got[:, 0]) == [30000, 60000 - 65536, 30000, 0]


@pytest.mark.parametrize("group", ["entropy", "header", "coef"])
def test_accepted_files_equal_imdecode_and_imdecode_refusals_are_refused(group):
    n_ok = 0
    for name, (b, edge) in _CASES.items():
        if (group == "header") != name.startswith("header/") or (group == "coef") != name.startswith("coef/"):
            continue
        want = imdecode(b)
        v = D.verdict(b)
        if want is None:
            assert v[0] != "ok", name
            continue
        if v[0] != "ok":
            continue
        got = R.decode(b)
        assert np.array_equal(got, want), name
        assert np.array_equal(R.bgr_to_gray(got), cv2.cvtColor(want, cv2.COLOR_BGR2GRAY)), name
        n_ok += 1
    assert n_ok > 0


def test_jpeg_info_gives_the_header_verdict():
    from denseflow_b200 import _lib, api
    for name, (b, edge) in _CASES.items():
        if not name.startswith("header/") and not name.endswith(("flip@0.0", "cut@7", "/no_eoi", "rst_deleted")):
            continue
        try:
            R.parse(b)
            want = ("ok", None)
        except R.Unsupported as e:
            want = (_lib.DFB_ERR_UNSUPPORTED, str(e))
        except R.Corrupt as e:
            want = (_lib.DFB_ERR_INVALID_ARG, str(e))
        L = _lib.load("default")
        import ctypes as C
        w, h = C.c_int(), C.c_int()
        buf = np.frombuffer(b, np.uint8)
        rc = L.dfb_jpeg_info(buf.ctypes.data, buf.size, C.byref(w), C.byref(h))
        if want[0] == "ok":
            hd = R.parse(b)
            assert rc == _lib.DFB_OK and (w.value, h.value) == (hd["w"], hd["h"]), name
            assert api.jpeg_info(b) == (hd["w"], hd["h"])
        else:
            assert rc == want[0], name
            assert L.dfb_last_error(None).decode() == "frame 0: " + want[1], name


def _fdct_extremes():
    """Per natural position, the least and greatest jpeg_fdct_islow output over every 8-bit block.  Each row's pass-1 output
    u is a descaled linear form of the row, extreme at one of the 256 rows of 0 / 255 samples; pass 2 is a descaled linear
    form of a column of 8 pass-1 outputs, one per row, which take their extremes independently, so it too is extreme at one of
    the 256 columns built from each row's least or greatest output.  Both descales are monotone."""
    verts = np.array([[127 if (m >> i) & 1 else -128 for i in range(8)] for m in range(256)], np.int64)
    p1 = E._fdct_1d(verts, True)
    lo1, hi1 = p1.min(0), p1.max(0)
    lo, hi = np.zeros(64, np.int64), np.zeros(64, np.int64)
    sel = np.array([[(m >> r) & 1 for r in range(8)] for m in range(256)], bool)
    for u in range(8):
        o = E._fdct_1d(np.where(sel, hi1[u], lo1[u]), False)
        lo[u::8], hi[u::8] = o.min(0), o.max(0)
    return lo, hi


def test_out_of_range_bound_covers_every_encoder_output():
    lo, hi = _fdct_extremes()
    # the extremes are reached: a flat block of 0 gives the DC minimum
    assert lo[0] == E.fdct(np.zeros((1, 8, 8), np.uint8))[0, 0] == -8192
    # over a brute-force sample of blocks, no output passes the extremes
    rng = np.random.default_rng(0)
    f = E.fdct(rng.choice(np.array([0, 255], np.uint8), (4096, 8, 8)))
    assert (f >= lo).all() and (f <= hi).all()
    # libjpeg-turbo's quantiser is monotone in |x|: the largest |q x quantised| at every 8- or 16-bit table entry
    qs = np.arange(1, 65536, dtype=np.int64)
    rc = np.array([E.reciprocal(int(q) << 3) for q in qs], np.int64)
    worst = 0
    for k in range(64):
        m = max(int(hi[k]), -int(lo[k]))
        c = ((m + rc[:, 1]) * rc[:, 0]) >> rc[:, 2]
        worst = max(worst, int((c * qs).max()))
    assert worst == R.MAX_DEQUANT
    # the quantiser restatement agrees with the division it stands for at the extremes
    assert E.quantize(np.full((1, 64), 8192), np.full(64, 2048))[0, 0] == 1


def test_out_of_range_bound_is_where_imdecode_stops_agreeing():
    """Single-coefficient blocks at every position: imdecode and the restatement's C IDCT agree up to the bound, and in
    every position class they part somewhere past it (so the bound is not looser than it has to be per class by much)."""
    q1 = np.ones(64, np.int64)

    def agree(k, v):
        blk = np.zeros((1, 64), np.int64)
        blk[0, k] = v
        b = D.write(8, 8, "gray", blk, q=q1, qbits=16)
        hd = R.parse(b)
        coef = R.coefficients(hd)
        try:
            return np.array_equal(R.to_bgr(hd, R.idct_planes(hd, coef)), imdecode(b))
        except R.Corrupt:  # an output past -512..511: refused
            return False

    first = {}
    for k in range(64):
        for v in (R.MAX_DEQUANT, -R.MAX_DEQUANT, 1024, -1024):
            assert agree(k, v), (k, v)
        first[k] = next((v for v in range(R.MAX_DEQUANT + 64, 32768, 64) if not (agree(k, v) and agree(k, -v))), None)
    assert all(v is not None and v > R.MAX_DEQUANT for v in first.values()), first
    assert min(first.values()) <= 2 * R.MAX_DEQUANT


def test_existing_fixtures_stay_inside_the_bound():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_decode_cases.npz"))
    for i in range(int(g["n"])):
        hd = R.parse(g["jpg%d" % i].tobytes())
        R.check_range(hd, R.coefficients(hd))


def test_huffman_refuses_a_code_of_all_ones():
    with pytest.raises(R.Corrupt, match="bad Huffman table"):
        R.Huffman([2] + [0] * 15, [0, 1], True)
    with pytest.raises(R.Corrupt, match="bad Huffman table"):
        R.Huffman([0, 0, 8] + [0] * 13, list(range(8)), False)
    R.Huffman([1, 1] + [0] * 14, [0, 1], True)  # "0", "10": "11" stays free
