"""Video-list dispatch on the GPU: several workers drain one dynamic queue; every video's outputs equal what a single
engine handle computes for it, chunks carry global flow indices, and `last_chunk` (the reference's
FlowBuffer::last_buffer, the only point where a .done marker may be written: /root/reference/src/denseflow_gpu.cpp:456-470)
fires exactly once per video, after all of its flows."""
import threading

import numpy as np
import pytest

from denseflow_b200 import listrun, synth

pytestmark = pytest.mark.gpu


def _clips():
    lens = [9, 1, 5, 12, 2, 7, 3]  # includes a one-frame video (no flow) and short ones
    return [list(synth.stream(96, 128, n, seed=200 + i, phase=3.0 * i)) for i, n in enumerate(lens)]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_list_outputs_match_single_handle(alg):
    import denseflow_b200 as d
    clips = _clips()
    e = d.create(alg, 0, 128, 96)
    want = [e.calc_batch(c, step=1, bound=20) if len(c) > 1 else (np.empty((0, 96, 128), np.uint8),) * 2 for c in clips]
    got = {i: {} for i in range(len(clips))}
    events = []
    lock = threading.Lock()

    def on_chunk(clip, dev, first, last, qx, qy, flows):
        with lock:
            assert flows is None
            for k in range(len(qx)):
                got[clip][first + k] = (qx[k].copy(), qy[k].copy())
            events.append((clip, first, len(qx), last, threading.get_ident()))

    st = listrun.run_list(alg, [0, 0, 0], clips, step=1, bound=20, chunk_flows=4, on_chunk=on_chunk)
    assert st["clips"] == len(clips) and st["flows"] == sum(max(len(c) - 1, 0) for c in clips)
    assert st["frames"] == sum(len(c) for c in clips) and sum(st["clips_per_worker"]) == len(clips)
    for i, c in enumerate(clips):
        m = max(len(c) - 1, 0)
        assert sorted(got[i]) == list(range(m))
        for j in range(m):
            assert np.array_equal(got[i][j][0], want[i][0][j]) and np.array_equal(got[i][j][1], want[i][1][j]), (i, j)
        ev = [x for x in events if x[0] == i]
        assert [x[3] for x in ev].count(True) == 1 and ev[-1][3]      # done exactly once, on the video's last chunk
        assert [x[1] for x in ev] == list(range(0, max(m, 1), 4))      # chunks of 4 flows, global first_flow indices
        assert len({x[4] for x in ev}) == 1                            # all from the worker that took the video


def test_list_float_flows_and_negative_step():
    import denseflow_b200 as d
    clips = _clips()[:4]
    e = d.create("tvl1", 0, 128, 96)
    got = {}

    def on_chunk(clip, dev, first, last, qx, qy, flows):
        assert qx is None
        for k in range(len(flows)):
            got[(clip, first + k)] = flows[k].copy()

    st = listrun.run_list("tvl1", [0, 0], clips, step=-2, bound=0, chunk_flows=3, on_chunk=on_chunk)
    for i, c in enumerate(clips):
        want = e.calc_batch(c, step=-2)
        assert want.shape[0] == max(len(c) - 2, 0)
        for j in range(want.shape[0]):
            assert np.array_equal(got[(i, j)], want[j]), (i, j)
    assert st["flows"] == sum(max(len(c) - 2, 0) for c in clips)


def test_two_workers_on_one_gpu_many_lanes():
    """BASELINE.json configs[4] shape (340x256x64) with two workers on ONE device: the 36-lane launches of the two handles
    overlap; every flow equals the single-handle result.  Regression test for the convergence-partial race that
    desynchronised the lane barrier under exactly this load."""
    import denseflow_b200 as d
    base = [list(synth.stream(256, 340, 64, seed=900 + i, phase=2.0 * i)) for i in range(2)]
    clips = [base[i % 2] for i in range(16)]
    e = d.create("tvl1", 0, 340, 256)
    want = [e.calc_batch(c, step=1, bound=32) for c in base]
    bad = []
    lock = threading.Lock()

    def on_chunk(clip, dev, first, last, qx, qy, flows):
        w = want[clip % 2]
        for k in range(len(qx)):
            if not (np.array_equal(qx[k], w[0][first + k]) and np.array_equal(qy[k], w[1][first + k])):
                with lock:
                    bad.append((clip, first + k))

    st = listrun.run_list("tvl1", [0, 0], clips, step=1, bound=32, on_chunk=on_chunk)
    assert st["flows"] == 16 * 63 and not bad, bad[:5]
