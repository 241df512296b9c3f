"""The GPU JPEG decoder on damaged and hand-built files (tests/jpeg_damage_cases.py), in both builds: a file the restatement
refuses is refused with the same DFB code and kind, naming its frame in a batch of good files; a file it accepts decodes to
its pixels and coefficients; the handle decodes good files right after every refusal."""
import ctypes as C

import cv2
import numpy as np
import pytest

import jpeg_cases as J
import jpeg_damage_cases as D
import jpeg_restate as R

pytestmark = pytest.mark.gpu
_handles = {}
_CASES = D.all_cases()
_VERDICTS = {name: D.verdict(b) for name, (b, _) in _CASES.items()}


def handle(variant="default", alg="tvl1", size=(1920, 1080)):
    import denseflow_b200 as d
    key = (variant, alg, size)
    if key not in _handles:
        _handles[key] = d.create(alg, 0, size[0], size[1], variant=variant)
    return _handles[key]


def raw_decode(e, files, mw=64, mh=64):
    """dfb_decode_jpeg_batch_device straight: (rc, last error, frames)"""
    import torch
    keep, ptrs, lens = e._jpeg_buffers(files)
    out = torch.zeros((len(files), mh, mw * 3), dtype=torch.uint8, device="cuda")
    rc = e._L.dfb_decode_jpeg_batch_device(e._h, ptrs, lens, len(files), 3, out.data_ptr(), mw * 3, mh * mw * 3, mw, mh, None, None, None)
    torch.cuda.synchronize()
    return rc, (e._L.dfb_last_error(e._h) or b"").decode(), out.cpu().numpy()


def decode(e, files, channels=3):
    import torch
    out = e.decode_jpeg_batch(files, channels)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


GOOD = [J.encode(J.image("noise", 37, 45), "420", 90), J.encode(J.image("smooth", 16, 61), "gray", 80, restart=2)]


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_refusals_name_the_frame_and_kind(variant):
    from denseflow_b200 import _lib
    e = handle(variant)
    want_good = [cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) for b in GOOD]
    refused = [n for n, v in _VERDICTS.items() if v[0] != "ok"]
    assert len(refused) > 1000
    for i, name in enumerate(refused):
        b = _CASES[name][0]
        k = i % 3
        files = GOOD[:k] + [b] + GOOD[k:]
        rc, msg, _ = raw_decode(e, files)
        v = _VERDICTS[name]
        assert rc == (_lib.DFB_ERR_UNSUPPORTED if v[0] == "unsupported" else _lib.DFB_ERR_INVALID_ARG), (name, rc, msg)
        assert msg.startswith("frame %d: " % k), (name, msg)
        assert D.kind(msg) == v[1], (name, msg, v)
        if i % 97 == 0:
            for got, w in zip(decode(e, GOOD), want_good):
                assert np.array_equal(got, w), name


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_accepted_files_give_the_restatements_pixels(variant):
    e = handle(variant)
    names = [n for n, v in _VERDICTS.items() if v[0] == "ok"]
    assert len(names) > 1000
    for s in range(0, len(names), 256):
        chunk = names[s:s + 256]
        files = [_CASES[n][0] for n in chunk]
        got, gray = decode(e, files, 3), decode(e, files, 1)
        for n, g, gg in zip(chunk, got, gray):
            want = R.decode(_CASES[n][0])
            assert np.array_equal(g, want), n
            assert np.array_equal(gg, R.bgr_to_gray(want)), n


def test_coefficients_equal_the_restatement():
    """Every file whose entropy decode succeeds (accepted, or refused only for out-of-range values): run-past-63 placement,
    the int16 DC wrap and in-range damage."""
    e = handle()
    n = 0
    for name, v in _VERDICTS.items():
        if v[0] != "ok" and v != ("corrupt", "range"):
            continue
        if name.startswith(("gray16/", "420_ri0/flip", "444_ri1/cut")) and n > 600:
            continue  # a sample of the large groups
        b = _CASES[name][0]
        got, _ = e.debug_jpeg_coefficients(b)
        want = R.coefficients(R.parse(b))
        assert np.array_equal(got.astype(np.int64), want), name
        n += 1
    assert n > 500


def test_large_damaged_file_then_small_good_one():
    from denseflow_b200 import _lib
    e = handle()
    big = J.encode(J.image("noise", 1080, 1920), "420", 95, restart=4)
    r = D.rst_positions(big)
    damaged = [big[:len(big) // 2] + b"\xff\xd9", big[:r[100]] + big[r[100] + 2:],
               big[:r[7] + 2] + b"\xff\x00" * 8 + big[r[7] + 2:]]
    for b in damaged:
        v = D.verdict(b)
        assert v[0] == "corrupt"
        with pytest.raises(RuntimeError) as ex:
            e.decode_jpeg_batch([GOOD[0], b])
        assert str(ex.value).count("frame 1") and D.kind(str(ex.value).split("frame 1: ", 1)[1]) == v[1], (str(ex.value), v)
        assert np.array_equal(decode(e, [GOOD[1]])[0], R.decode(GOOD[1]))
    assert D.verdict(damaged[2]) == ("corrupt", "code")
    rc, _, _ = raw_decode(e, [damaged[0]], 1920, 1080)
    assert rc == _lib.DFB_ERR_INVALID_ARG


def test_damaged_frame_in_the_second_group_of_a_chain():
    from denseflow_b200 import synth
    e = handle("default", "tvl1", (96, 64))
    gray = synth.stream(64, 96, 19, seed=4)
    files = [J.encode(np.stack([g, g, 255 - g], -1).astype(np.uint8), "420", 95) for g in gray]
    good = e.process_jpeg_batch(files, 1, 20)
    for bad in (files[13][:len(files[13]) // 2] + b"\xff\xd9", D._flip(files[13], D.scan_span(files[13])[0] + 3, 7)):
        if D.verdict(bad)[0] == "ok":
            continue
        with pytest.raises(RuntimeError, match="frame 13"):
            e.process_jpeg_batch(files[:13] + [bad] + files[14:], 1, 20)
        assert e.process_jpeg_batch(files, 1, 20) == good
