"""Both engines at the geometries of tests/geometry_cases.py, through every entry point of the C ABI.

At every frame size, for TV-L1 and Farneback, in both builds:
* the flow of dfb_calc_host is pinned to the oracle: bit for bit with the same iteration schedule in the strict build
  (tests/tvl1_pin.py decides borderline convergence checks), within the 0.01 px contract and finite in the default build;
* every other entry point gives the same bytes as dfb_calc_host on the same handle: dfb_calc_batch_host and
  dfb_calc_batch_host_u8 with pageable and with page-locked frames and outputs, dfb_calc_device on dense tensors, on pitched
  views whose base is 1 to 3 bytes off alignment and on a stream of its own, and dfb_calc_batch_device at steps +-1 and
  +-3, with no pair at all and with more pairs than one launch takes (TV-L1 at 2 lanes, Farneback's 8 pairs per launch).
One handle per algorithm and build, created at 3840 x 2160, serves the sweep from 4K down to 1 x 1 (the workspace, the frame
slots and the tensor maps are re-targeted at every size); handles created at tiny maximum sizes serve the frames that fit.
Host and device entry points are never in flight on one handle at the same time: every device call is synchronised."""
import numpy as np
import pytest

import geometry_cases as gc
import tvl1_pin as pin
from denseflow_b200 import synth

pytestmark = pytest.mark.gpu
VARIANTS = ["strict", "default"]
ALGORITHMS = ["tvl1", "farn"]
AEE_TOL = 0.01  # px, BASELINE.json north_star
BOUND = 20
STEPS = (1, -1, 3, -3)
_handles = {}
_oracle = {}


def _handle(alg, variant, w=3840, h=2160):
    key = (alg, variant, w, h)
    if key not in _handles:
        import denseflow_b200 as d
        _handles[key] = d.create(alg, 0, w, h, variant)
    return _handles[key]


def _frames(w, h):
    """10 frames (9 pairs at step 1: two Farneback launches, five TV-L1 launches at 2 lanes); 4 above one megapixel"""
    return synth.stream(h, w, 10 if w * h <= 1 << 20 else 4, seed=7 * w + h)


def _batches(fr):
    """(step, frames) of the batches: step 1 over all frames, the other steps over the first six"""
    return [(step, fr if step == 1 else fr[:6]) for step in STEPS]


def _pairs(step, n):
    """(first, second) frame of every pair of a batch (src/denseflow_gpu.cpp:315-316)"""
    a = abs(step)
    return [(j, j + a) if step > 0 else (j + a, j) for j in range(max(n - a, 0))]


def _oracle_out(oracle, alg, fr):
    """the oracle's flow (and TV-L1 log and convergence checks) of frames 0 -> 1, shared by the two builds"""
    key = (alg, fr.shape, fr[0].tobytes()[:64])
    if key not in _oracle:
        _oracle.clear()
        big = fr[0].size > 1 << 20
        if big:
            oracle.lib().orc_set_num_threads(oracle.usable_cores())
        try:
            _oracle[key] = (oracle.tvl1_calc(fr[0], fr[1], return_iters=True, return_errors=True) if alg == "tvl1"
                            else (oracle.farn_calc(fr[0], fr[1]),))
        finally:
            if big:
                oracle.lib().orc_set_num_threads(min(8, oracle.usable_cores()))
    return _oracle[key]


def _same(got, want, name):
    diff = np.any(got != want, axis=-1) if got.ndim == 3 else got != want
    assert not diff.any(), "%s: %d pixels differ from calc_host, first at %s" % (name, diff.sum(), tuple(np.argwhere(diff)[0]))


def _pin_to_oracle(oracle, e, alg, variant, fr, flow, iters, tag):
    """None, or the note of a borderline TV-L1 convergence check (strict build)"""
    out = _oracle_out(oracle, alg, fr)
    ref = out[0]
    assert np.isfinite(flow).all(), tag
    # the quantised planes are the CAST of the flow (which the strict build pins to the oracle's below)
    qx, qy = e.calc_batch(list(fr[:2]), step=1, bound=BOUND)
    ox, oy = oracle.quantise(flow, BOUND)
    _same(qx[0], ox, tag + " qx")
    _same(qy[0], oy, tag + " qy")
    if variant == "default":
        aee = synth.aee(flow, ref)
        assert aee <= AEE_TOL, (tag, aee)
        return None
    if alg == "tvl1":
        return pin.check(oracle, fr[0], fr[1], flow, iters, tag, oracle_out=out)
    diff = np.any(flow != ref, axis=-1)
    assert not diff.any(), "%s: %d pixels differ from orc_farn_calc, first at %s" % (tag, diff.sum(), tuple(np.argwhere(diff)[0]))
    return None


class _Host:
    """dfb_calc_host of frame pairs on one handle, each pair computed once"""

    def __init__(self, e, fr):
        self.e, self.fr, self.done = e, fr, {}

    def __call__(self, i, k):
        if (i, k) not in self.done:
            self.done[(i, k)] = self.e.calc(self.fr[i], self.fr[k])
        return self.done[(i, k)]


def _host_batches(e, fr, host, tag):
    """pageable frames and outputs at every step (staged through the handle's pinned ring); page-locked frames and outputs
    (direct copies) at steps 1 and -3; the quantised planes into pageable arrays at step -1, into page-locked ones at step 3"""
    import torch
    h, w = fr.shape[1:]
    pinned = torch.from_numpy(fr).pin_memory().numpy()
    for step, frs in _batches(fr):
        ps = _pairs(step, len(frs))
        flows = e.calc_batch(list(frs), step=step)
        assert flows.shape[0] == len(ps)
        for j, (a, b) in enumerate(ps):
            _same(flows[j], host(a, b), "%s calc_batch_host step %d pair %d" % (tag, step, j))
        if step in (1, -3):
            out = torch.empty((len(ps), h, w, 2), dtype=torch.float32).pin_memory().numpy()
            e.calc_batch(list(pinned[:len(frs)]), step=step, flows=out)
            for j, (a, b) in enumerate(ps):
                _same(out[j], host(a, b), "%s calc_batch_host pinned step %d pair %d" % (tag, step, j))
        else:
            if step == -1:
                qx, qy = e.calc_batch(list(frs), step=step, bound=BOUND)
                kind = "pageable"
            else:
                qx = torch.empty((len(ps), h, w), dtype=torch.uint8).pin_memory().numpy()
                qy = torch.empty((len(ps), h, w), dtype=torch.uint8).pin_memory().numpy()
                e.calc_batch_u8_into(list(pinned[:len(frs)]), step, BOUND, qx, qy)
                kind = "pinned"
            for j, (a, b) in enumerate(ps):
                ox, oy = _quantise(host(a, b))
                _same(qx[j], ox, "%s calc_batch_host_u8 %s step %d pair %d qx" % (tag, kind, step, j))
                _same(qy[j], oy, "%s calc_batch_host_u8 %s step %d pair %d qy" % (tag, kind, step, j))
    assert e.calc_batch(list(fr[:3]), step=3).shape[0] == 0
    assert e.calc_batch(list(pinned[:2]), step=-3, bound=BOUND)[0].shape[0] == 0


def _quantise(flow):
    from oracle import pyoracle
    return pyoracle.quantise(flow, BOUND)


def _device_calls(e, alg, fr, host, tag):
    import torch
    n, h, w = fr.shape
    dfr = torch.from_numpy(fr).cuda()
    want = host(0, 1)
    got = e.calc(dfr[0], dfr[1])
    torch.cuda.synchronize()
    _same(got.cpu().numpy(), want, tag + " calc_device dense")
    # pitched views whose base is 1..3 bytes past an aligned address (the uchar4 loads of k_u8_to_f32_batch must not be taken),
    # into a flow whose rows are longer than the image
    for off in (1, 2, 3):
        pitch = w + 8 + 2 * off + 1
        buf = torch.zeros((2, h * pitch + off), dtype=torch.uint8, device="cuda")
        va, vb = (buf[k, off:off + h * pitch].view(h, pitch)[:, :w] for k in (0, 1))
        va.copy_(dfr[0])
        vb.copy_(dfr[1])
        flow = torch.full((h, w + 3, 2), float("nan"), dtype=torch.float32, device="cuda")[:, :w]
        assert va.data_ptr() % 4 == off and va.stride(0) == pitch
        e.calc(va, vb, flow=flow)
        torch.cuda.synchronize()
        _same(flow.cpu().numpy(), want, "%s calc_device base +%d pitch %d" % (tag, off, pitch))
    # on a stream of its own
    s = torch.cuda.Stream()
    out = torch.full((h, w, 2), float("nan"), dtype=torch.float32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    e.calc(dfr[0], dfr[1], flow=out, stream=s.cuda_stream)
    s.synchronize()
    _same(out.cpu().numpy(), want, tag + " calc_device on another stream")
    # batches on the device: TV-L1 at 2 lanes, so that a batch takes several launches and the frame slots are reused
    if alg == "tvl1":
        e.set("lanes", 2)
    try:
        for step, frs in _batches(fr):
            ps = _pairs(step, len(frs))
            flows = e.calc_batch_device(dfr[:len(frs)], step=step)
            torch.cuda.synchronize()
            assert flows.shape[0] == len(ps)
            got = flows.cpu().numpy()
            for j, (a, b) in enumerate(ps):
                _same(got[j], host(a, b), "%s calc_batch_device step %d pair %d" % (tag, step, j))
        for k, step in ((1, 1), (3, -3), (2, 3)):  # n_frames <= |step|: no pair, nothing written
            assert e.calc_batch_device(dfr[:k].contiguous(), step=step).shape[0] == 0
        torch.cuda.synchronize()
    finally:
        if alg == "tvl1":
            e.set("lanes", 0)


def _e2e_ids():
    return ["%s-%dx%d" % (alg, w, h) for alg in ALGORITHMS for w, h in gc.e2e(alg)]


@pytest.mark.parametrize("variant", VARIANTS)  # the top parameter varies fastest: both builds share one oracle run per case
@pytest.mark.parametrize("case", [(alg, s) for alg in ALGORITHMS for s in gc.e2e(alg)], ids=_e2e_ids())
def test_every_entry_point_at_every_geometry(oracle, case, variant):
    alg, (w, h) = case
    e = _handle(alg, variant)
    fr = _frames(w, h)
    host = _Host(e, fr)
    tag = "%s %s %dx%d" % (alg, variant, w, h)
    flow = host(0, 1)
    iters = e.tvl1_stats()[0] if alg == "tvl1" else None
    note = _pin_to_oracle(oracle, e, alg, variant, fr, flow, iters, tag)
    _host_batches(e, fr, host, tag)
    if alg == "tvl1":  # groups of 2 pairs: a call of 5 or more pairs reuses the output slots of its two groups in flight
        e.set("lanes", 2)
        try:
            _host_batches(e, fr, host, tag + " lanes 2")
        finally:
            e.set("lanes", 0)
    _device_calls(e, alg, fr, host, tag)
    pin.finish([note])


TINY_MAX = [(1, 1), (3, 2), (1, 8), (8, 1), (13, 13), (33, 17)]


@pytest.mark.parametrize("alg", ALGORITHMS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_handles_created_at_tiny_sizes(oracle, variant, alg):
    """a handle whose maximum frame is tiny (workspace, slots and lanes sized for it) computes what the 4K handle computes, at
    its maximum size and at the smaller sweep sizes that fit it, on the host and on the device"""
    import torch
    big = _handle(alg, variant)
    for mw, mh in TINY_MAX:
        e = _handle(alg, variant, mw, mh)
        fits = [(mw, mh)] + [s for s in gc.e2e(alg) if s[0] <= mw and s[1] <= mh and s != (mw, mh)][:4]
        for w, h in fits:
            fr = _frames(w, h)[:5]
            tag = "%s %s handle %dx%d frame %dx%d" % (alg, variant, mw, mh, w, h)
            want = [big.calc(fr[j], fr[j + 1]) for j in range(4)]
            flows = e.calc_batch(list(fr), step=1)
            dev = e.calc_batch_device(torch.from_numpy(fr).cuda(), step=1)
            torch.cuda.synchronize()
            dev = dev.cpu().numpy()
            for j in range(4):
                _same(e.calc(fr[j], fr[j + 1]), want[j], "%s calc_host pair %d" % (tag, j))
                _same(flows[j], want[j], "%s calc_batch_host pair %d" % (tag, j))
                _same(dev[j], want[j], "%s calc_batch_device pair %d" % (tag, j))
    with pytest.raises(RuntimeError, match="exceeds"):
        _handle(alg, variant, 1, 1).calc(np.zeros((1, 2), np.uint8), np.zeros((1, 2), np.uint8))
