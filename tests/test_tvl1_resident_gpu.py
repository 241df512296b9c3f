"""Resident tiles of the fused TV-L1 kernel end to end.  A level with no more tiles than a lane has CTAs keeps them on chip
across the chunks of a warp's epoch loop: later chunks read back only the ring, write back only the band, and the last
chunk of every epoch writes the whole interior (tvl1_fused.cu, run_chunk).

* 1080p: 2 lanes (66 CTAs each: the 63 tiles of the coarsest level are resident), 4 lanes (33 CTAs: every level streams)
  and the unfused schedule give the same flows and iteration logs, in both builds;
* 340x256 and 256x256 on one lane (every level resident) equal the oracle bit for bit in the strict build, with epochs
  cut into chunks of mixed length (8, 8, 7 at 23 iterations; 2 and 3 at fused_k 3)."""
import numpy as np
import pytest

import tvl1_pin as pin
from denseflow_b200 import synth

pytestmark = pytest.mark.gpu


def _new(w, h, variant, **params):
    import denseflow_b200 as d
    e = d.OpticalFlowDual_TVL1.create(0, w, h, variant)
    for k, v in params.items():
        e.set(k, v)
    return e


@pytest.mark.parametrize("variant", ["strict", "default"])
def test_1080p_resident_and_streamed_agree(variant):
    h, w = 1080, 1920
    fr = list(synth.stream(h, w, 5, seed=1))
    runs = {}
    for name, params in (("lanes 2", {"lanes": 2}), ("lanes 4", {"lanes": 4}), ("unfused", {"fused": 0})):
        e = _new(w, h, variant, **params)
        flows = e.calc_batch(fr, step=1)
        logs = [e.tvl1_pair_stats(j).copy() for j in range(len(fr) - 1)]
        runs[name] = (flows, logs)
        e.release()
    ref_flows, ref_logs = runs["unfused"]
    for name in ("lanes 2", "lanes 4"):
        flows, logs = runs[name]
        for j in range(len(fr) - 1):
            assert np.array_equal(logs[j], ref_logs[j]), "%s pair %d: iteration log differs" % (name, j)
            diff = np.any(flows[j] != ref_flows[j], axis=-1)
            assert not diff.any(), "%s %s pair %d: %d pixels differ from the unfused schedule, first at %s" % (
                variant, name, j, diff.sum(), tuple(np.argwhere(diff)[0]))


CASES = [((256, 340), {}), ((256, 256), {}), ((256, 340), {"epsilon": 0.0, "iterations": 23}), ((256, 256), {"fused_k": 3}),
         ((256, 340), {"warps": 2, "iterations": 37})]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_every_level_resident_is_bit_exact(oracle, case):
    (h, w), params = CASES[case]
    fr = synth.stream(h, w, 3, seed=20 + case)
    e = _new(w, h, "strict", lanes=1, **params)
    op = {k: v for k, v in params.items() if k in ("nscales", "warps", "iterations", "epsilon")}
    flows = e.calc_batch(list(fr), step=1)
    notes = [pin.check(oracle, fr[j], fr[j + 1], flows[j], e.tvl1_pair_stats(j), "%dx%d %s pair %d" % (w, h, params, j),
                       oracle.tvl1_params(**op)) for j in range(len(fr) - 1)]
    pin.finish(notes)
