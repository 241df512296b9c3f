"""zlib's deflate edges that the GPU PNG encoder restates (denseflow_b200/csrc/png_deflate.cuh), on content built to reach
them (tests/deflate_cases.py): every case is checked to reach its edge in zlib's own stream, the restatement equals
cv2.imencode on it, the size model (tests/zlib_sizes.py) equals zlib on every block, and a host build of the encoder's
per-block code (tests/pngz_host_shim.cpp) equals zlib block by block: type, code lengths, header bits and block bits."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import deflate_cases as D
import inflate_trace as T
import png_cases as PC
import png_restate as P
import zlib_sizes as Z

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "denseflow_b200", "csrc")

_cases = {}


def cases():
    if not _cases:
        _cases.update((n, (img, edge)) for n, img, edge in D.cases())
    return _cases


NAMES = [n for n, _, _ in D.cases()]


def _trace(img):
    raw = P.scanlines(img)
    z = P.zlib_stream(raw)
    blocks, data = T.trace(z)
    assert data == raw
    return raw, z, blocks


def _model_equals_zlib(raw, tblocks):
    """the size model gives zlib's block types on every block, its code lengths on dynamic blocks and its bit counts on
    fixed and dynamic ones"""
    mblocks = Z.blocks(raw)
    assert len(mblocks) == len(tblocks)
    for i, (t, m) in enumerate(zip(tblocks, mblocks)):
        assert t["type"] == m["type"], (i, t["type"], m["type"], m["stored_len"], m["dyn_lenb"], m["static_lenb"])
        if t["type"] == "stored":
            assert t["stored_len"] == m["stored_len"], i
            continue
        assert t["end"] - t["start"] == m["bits"], i
        if t["type"] == "dynamic":
            assert t["lit_lengths"] == m["lit"]["lengths"][:m["lit"]["max_code"] + 1], i
            assert t["dist_lengths"] == m["dist"]["lengths"][:m["dist"]["max_code"] + 1], i
            assert t["code_lengths"] == m["bl"]["lengths"], i
    return mblocks


def _edge(name, raw, z, tb, mb):
    """asserts that the case reaches the edge it was built for"""
    b0 = mb[0]
    if name.startswith(("fibonacci", "lucas")):
        d = int(name.lstrip("abcfilnosu"))
        assert len(mb) == 1 and b0["type"] == "dynamic" and b0["lit"]["depth"] == d and b0["lit"]["overflow"] > 0
        assert max(tb[0]["lit_lengths"]) == 15
    elif name == "deep_middle_block":
        assert [b["type"] for b in mb] == ["stored", "dynamic", "stored"] and not tb[1]["final"]
        assert mb[1]["lit"]["depth"] == 17 and mb[1]["lit"]["overflow"] > 0 and mb[0]["lit"]["overflow"] == mb[2]["lit"]["overflow"] == 0
    elif name == "deep_with_lengths":
        assert len(mb) == 1 and b0["type"] == "dynamic" and b0["lit"]["depth"] == 17 and b0["lit"]["overflow"] > 0
        for code, lens in D.CHAIN_MATCHES.items():
            assert b0["lfreq"][code] == len(lens) and Z.EXTRA_LBITS[code - 257] > 0
            assert tb[0]["lit_lengths"][code] == 15  # repaired: deeper than 15 before
        assert sorted(s[0] for s in tb[0]["symbols"] if isinstance(s, tuple)) == sorted(n for v in D.CHAIN_MATCHES.values() for n in v)
    elif name.startswith("geometric"):
        assert len(mb) == 1 and b0["type"] == "dynamic" and b0["bl"]["depth"] >= 8 and b0["bl"]["overflow"] > 0
        assert max(tb[0]["code_lengths"]) == 7
    elif name.startswith("only_literal"):
        v = int(name[-1])
        assert all([i for i in range(256) if b["lfreq"][i]] == [v] for b in mb)
        assert all(b["dist"]["fake"] == [1] and b["dfreq"][0] > 0 for b in mb)
    elif name == "no_matches":
        assert b0["type"] == "dynamic" and b0["dist"]["fake"] == [0, 1] and b0["dfreq"][0] == 0
    elif name == "empty_final_block":
        assert mb[-1]["nsym"] == 0 and mb[-1]["lit"]["fake"] == [0] and mb[-1]["lit"]["max_code"] == 256
        assert tb[-1]["type"] == "fixed" and tb[-1]["symbols"] == []
    elif name.startswith("stored+"):
        k = int(name[len("stored+"):])
        assert len(mb) == 1 and min(b0["dyn_lenb"], b0["static_lenb"]) == b0["stored_len"] + k
        assert b0["type"] == ("stored" if k >= 4 else "fixed" if b0["static_lenb"] <= b0["dyn_lenb"] else "dynamic")
        # zlib's own min(dynamic, fixed) size of this histogram: the same block with its one match 6 bytes longer (the same
        # length code) covers 6 more bytes, so zlib no longer stores it and its bit count shows the size
        params = dict(D.STORED_TIES)[name]
        raw6, _, tb6 = _trace(D.stretched_run_noise(*params, stretch=6))
        m6 = _model_equals_zlib(raw6, tb6)
        assert len(tb6) == 1 and tb6[0]["type"] != "stored" and m6[0]["stored_len"] == b0["stored_len"] + 6
        assert (m6[0]["lfreq"], m6[0]["dfreq"]) == (b0["lfreq"], b0["dfreq"])
        assert (tb6[0]["end"] - tb6[0]["start"] + 7) >> 3 == b0["stored_len"] + k
    elif name.startswith("fixed=dynamic"):
        k = int(name[len("fixed=dynamic"):])
        assert len(mb) == 1 and b0["static_lenb"] == b0["dyn_lenb"] + k and b0["stored_len"] + 4 > min(b0["static_lenb"], b0["dyn_lenb"])
        assert b0["type"] == ("fixed" if k <= 0 else "dynamic")
    elif name.startswith("flush_at_run_"):
        code, lens = Z.symbols(raw)
        run0 = raw.index(b"\x07" * 777)
        pos = int(np.sum(lens[:16382]))  # first byte of the block's last symbol
        where = name[len("flush_at_run_"):]
        assert run0 <= pos < run0 + 777
        if where == "head":
            assert pos == run0 and code[16382] == 7 and code[16383] == 285
        elif where == "match":
            assert pos == run0 + 1 + 258 and code[16382] == 285 and code[16381] == 285 and code[16383] == 285
        else:
            assert pos == run0 + 1 + 3 * 258 and code[16382] == 7 and code[16381] == 285 and code[16383] == 7
        assert len(mb) >= 2 and mb[0]["nsym"] == 16383
    elif name.startswith("window_"):
        n = len(raw)
        k, d, w1 = re.fullmatch(r"window_2\^(\d+)([+-]\d+)?( w1)?", name).groups()
        assert n == (1 << int(k)) + int(d or 0) and raw[0] == (0 if w1 else 1)  # filter NONE only at width 1
        cinfo = z[0] >> 4
        assert (1 << (cinfo + 8)) >= n and (cinfo == 0 or (1 << (cinfo + 7)) < n)
        if n & (n - 1) == 0:
            assert 1 << (cinfo + 8) == n  # the declared window is exactly the data
    elif name.startswith("idat_"):
        t = int(name[len("idat_"):])
        assert len(z) == t
    else:
        raise AssertionError(name)


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_edge(name):
    img, _ = cases()[name]
    raw, z, tb = _trace(img)
    mb = _model_equals_zlib(raw, tb)
    _edge(name, raw, z, tb, mb)


def test_chain_depths_around_the_limits():
    """A chain 15 deep needs no repair.  Four 1s collapse the chain (they pair into two nodes of 2), which is why the
    filter byte and END_BLOCK are the Fibonacci chain's only 1s.  The Lucas chain is 18 deep in a 9 349-byte stream where
    the Fibonacci chain needs 10 944, and 19 deep in 15 127 (lucas19).  No block can be 20 deep: a Huffman tree with a
    leaf at depth d and least weight 1 weighs at least F(d + 2), 17 711 for d = 20, more than the 16 384 (END_BLOCK
    included) of a block.  At depth 20 the Lucas stream takes two blocks, and neither needs a repair."""
    raw, _, tb = _trace(D.fibonacci(15))
    m = Z.blocks(raw)[0]
    assert m["lit"]["depth"] == 15 and m["lit"]["overflow"] == 0 and max(tb[0]["lit_lengths"]) == 15
    counts = {1: 1}
    vals = D.chain_values(17)
    counts.update(zip(vals, [1, 1] + D.FIB[2:17]))
    w = D._fit_top(counts, vals[-1])
    raw, _, tb = _trace(D.literal_histogram(counts, 1, w))
    assert _model_equals_zlib(raw, tb)[0]["lit"]["depth"] < 15
    raw, _, tb = _trace(D.lucas(18))
    assert len(raw) == 9349 and _model_equals_zlib(raw, tb)[0]["lit"]["depth"] == 18
    raw, _, tb = _trace(D.lucas(20))
    mb = _model_equals_zlib(raw, tb)
    assert len(mb) == 2 and all(b["lit"]["overflow"] == 0 for b in mb)


def test_realistic_flow_needs_literal_repair():
    """the packed image of a smooth flow field plus 0.05 px noise, as -st=png writes it, has a block whose literal tree
    zlib repairs"""
    from oracle import cv_restate as R
    img, _, _ = R.flow_to_png_image(D.synthetic_flow())
    raw = P.scanlines(img)
    mb = Z.blocks(raw)
    assert any(b["type"] == "dynamic" and b["lit"]["overflow"] for b in mb)
    tb, data = T.trace(P.zlib_stream(raw))
    assert data == raw and [b["type"] for b in tb] == [b["type"] for b in mb]
    for t, m in zip(tb, mb):
        if m["lit"]["overflow"] and t["type"] == "dynamic":
            assert t["lit_lengths"] == m["lit"]["lengths"][:m["lit"]["max_code"] + 1]


def test_model_equals_zlib_on_png_cases():
    for kind in PC.CONTENTS:
        for h, w in PC.PROBE_SIZES:
            if h * w <= 256 * 340:
                img = PC.image(kind, h, w)
                raw, _, tb = _trace(img)
                _model_equals_zlib(raw, tb)
    for shape in PC.BLOCK_EDGE_SIZES:
        raw, _, tb = _trace(PC.literal_noise(*shape))
        _model_equals_zlib(raw, tb)
    for n in (3, 4, 258, 259, 260, 261, 517):
        raw, _, tb = _trace(PC.run_image(n))
        _model_equals_zlib(raw, tb)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_imencode(name):
    cv2 = pytest.importorskip("cv2")
    img, _ = cases()[name]
    ok, want = cv2.imencode(".png", img)
    assert ok
    got = P.encode(img)
    assert got == want.tobytes(), T.first_difference(P.idat_stream(got), P.idat_stream(want.tobytes()))


# ---- the encoder's block code, built for the host ----

@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "g++")) or shutil.which("c++")
    if not cxx:
        pytest.skip("no C++ compiler")
    out = str(tmp_path_factory.mktemp("pngz") / "pngz_host_shim.so")
    subprocess.run([cxx, "-std=c++17", "-O1", "-shared", "-fPIC", "-I", CSRC, os.path.join(HERE, "pngz_host_shim.cpp"), "-o", out],
                   check=True)
    lib = C.CDLL(out)
    lib.pngz_flush_block.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def flush_block(lib, lfreq, dfreq, stored_len, last):
    lf, df = np.array(lfreq, np.uint32), np.array(dfreq, np.uint32)
    out, sizes = np.zeros(5, np.uint32), np.zeros(2, np.int64)
    lit, tree, hdr = np.zeros(Z.L_CODES, np.uint32), np.zeros(Z.L_CODES, np.uint32), np.zeros(144, np.uint32)
    lib.pngz_flush_block(lf.ctypes.data, df.ctypes.data, stored_len, int(last), out.ctypes.data, sizes.ctypes.data, lit.ctypes.data,
                         tree.ctypes.data, hdr.ctypes.data)
    return {"type": ["stored", "fixed", "dynamic"][out[0]], "hdr_bits": int(out[1]), "bits": int(out[2]), "dist_len": int(out[3]),
            "opt_len": int(sizes[0]), "static_len": int(sizes[1]), "lit": lit.tolist(), "hdr": hdr, "lmax": int(out[4]),
            "tree": tree.tolist()}


def _bits(words_or_bytes, start, n, word_bits):
    """n bits from bit `start` of an LSB-first buffer of word_bits-bit units, as a 0/1 list"""
    return [(int(words_or_bytes[(start + i) // word_bits]) >> ((start + i) % word_bits)) & 1 for i in range(n)]


def _shim_equals_zlib(lib, img):
    raw, z, tb = _trace(img)
    mb = Z.blocks(raw)
    assert len(tb) == len(mb)
    for i, (t, m) in enumerate(zip(tb, mb)):
        g = flush_block(lib, m["lfreq"], m["dfreq"], m["stored_len"], t["final"])
        where = "block %d" % i
        assert g["type"] == t["type"], where
        # the sizes the choice is made from and the literal / length tree built, which a stored or fixed block does not show
        # (the empty final block's tree is END_BLOCK and the fake node build_tree adds at 0)
        assert (g["opt_len"], g["static_len"]) == (m["opt_len"], m["static_len"]), where
        assert (g["lmax"], g["tree"]) == (m["lit"]["max_code"], m["lit"]["lengths"]), where
        if t["type"] == "stored":
            continue
        assert g["bits"] == t["end"] - t["start"], where
        assert g["hdr_bits"] == t["body"] - t["start"], where
        assert _bits(g["hdr"], 0, g["hdr_bits"], 32) == _bits(z, t["start"], g["hdr_bits"], 8), where
        if t["type"] == "fixed":
            assert g["lit"] == [8] * 144 + [9] * 112 + [7] * 24 + [8] * 6 and g["dist_len"] == 5, where
            continue
        hlit = len(t["lit_lengths"])
        assert g["lit"][:hlit] == t["lit_lengths"] and not any(g["lit"][hlit:]), where
        assert g["dist_len"] == t["dist_lengths"][0], where
        # the code-length code lengths, read back from the header the shim wrote
        hb = _bits(g["hdr"], 0, g["hdr_bits"], 32)
        val = lambda p, n: sum(b << k for k, b in enumerate(hb[p:p + n]))  # noqa: E731
        hclen = val(13, 4) + 4
        cl = [0] * 19
        for r in range(hclen):
            cl[Z.BL_ORDER[r]] = val(17 + 3 * r, 3)
        assert cl == t["code_lengths"], where
    return mb


@pytest.mark.parametrize("name", NAMES)
def test_host_block_code_equals_zlib(shim, name):
    img, _ = cases()[name]
    _shim_equals_zlib(shim, img)


def test_host_block_code_on_png_cases(shim):
    for kind in PC.CONTENTS:
        for h, w in [(9, 9), (64, 64), (256, 340), (73, 74)]:
            _shim_equals_zlib(shim, PC.image(kind, h, w))
    for n in (3, 259, 517):
        _shim_equals_zlib(shim, PC.run_image(n))


def test_host_block_code_on_realistic_flow(shim):
    from oracle import cv_restate as R
    img, _, _ = R.flow_to_png_image(D.synthetic_flow())
    mb = _shim_equals_zlib(shim, img)
    assert any(b["lit"]["overflow"] for b in mb)


def test_max_bytes_bounds_every_case():
    from denseflow_b200 import _lib
    L = _lib.load("default")
    for name, (img, _) in cases().items():
        h, w = img.shape[:2]
        assert L.dfb_png_max_bytes(w, h) >= len(P.encode(img)), name
