"""GPU quantiser vs the CAST macro of /root/reference/src/common.cpp:6 (bit-exact)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_quantise_device_bit_exact(oracle):
    import torch
    import denseflow_b200 as d
    rng = np.random.default_rng(0)
    h, w = 77, 203
    flow = (rng.standard_normal((h, w, 2)) * 15).astype(np.float32)
    # ties: v = L + (k+0.5)(H-L)/255 for every k, clamps, exact bounds
    for bound in (20, 32, 7):
        k = np.arange(255)
        ties = (-bound + (k + 0.5) * (2 * bound) / 255).astype(np.float32)
        flow[0, :255 if w >= 255 else w, 0] = ties[:min(w, 255)]
        flow[1, :8, 1] = [-bound, bound, -bound - 1e-3, bound + 1e-3, 0, -0.0, 1e30, -1e30]
        e = d.OpticalFlowDual_TVL1.create(0, 256, 256)
        qx, qy = e.quantise_device(torch.from_numpy(flow).cuda(), bound)
        ox, oy = oracle.quantise(flow, bound)
        assert np.array_equal(qx.cpu().numpy(), ox)
        assert np.array_equal(qy.cpu().numpy(), oy)


def _decision_points(bound):
    """for each of the 255 values where 255 * (v + B) / 2B crosses k + 0.5: the float nearest it and one ulp either side"""
    k = np.arange(255)
    v = (-bound + (k + 0.5) * (2.0 * bound) / 255).astype(np.float32)
    return np.concatenate([np.nextafter(v, np.float32(-np.inf)), v, np.nextafter(v, np.float32(np.inf))])


@pytest.mark.parametrize("bound", [1, 20, 32])
@pytest.mark.parametrize("shape", [(1, 1), (1, 2000), (2000, 1), (3, 7)])
def test_quantise_decision_points_specials_and_pitch(oracle, shape, bound):
    """1 x 1, a single row, a single column; every decision point +-1 ulp, +-0, +-inf, NaN, the bounds and one ulp past
    them; a flow whose rows are longer than the image (pitch 8 w + 40 bytes)"""
    import torch
    import denseflow_b200 as d
    h, w = shape
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, bound, -bound, np.nextafter(np.float32(bound), np.float32(np.inf)),
                        np.nextafter(np.float32(-bound), np.float32(-np.inf))], np.float32)
    vals = np.concatenate([_decision_points(bound), special])
    e = d.OpticalFlowDual_TVL1.create(0, 64, 64)
    for start in range(0, len(vals), w * h):
        flat = np.resize(np.roll(vals, -start), 2 * w * h).astype(np.float32)
        flow = np.ascontiguousarray(np.stack([flat[:w * h], flat[::-1][:w * h]], -1).reshape(h, w, 2))
        dev = torch.full((h, w + 5, 2), float("nan"), dtype=torch.float32, device="cuda")[:, :w]
        dev.copy_(torch.from_numpy(flow))
        qx, qy = e.quantise_device(dev, bound)
        torch.cuda.synchronize()
        ox, oy = oracle.quantise(flow, bound)
        assert np.array_equal(qx.cpu().numpy(), ox) and np.array_equal(qy.cpu().numpy(), oy), (shape, bound, start)
        if w * h >= len(vals):
            break
