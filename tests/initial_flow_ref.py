"""The Farneback warm start (`use_initial_flow`, DESIGN §1) restated for the tests.  The oracle's own entry point stays as it
is; `farn_calc` restates orc_farn_calc's level loop over the C Farneback building blocks, with the coarsest level starting
from `farn_start`: orc_resize_linear(initial flow) to its size (explicit size, the oracle's resize convention) times
float(pyr_scale^k).  With a zero initial flow it is orc_farn_calc bit for bit (tests/test_initial_flow_cpu.py checks that).
The TV-L1 warm start is restated in tests/tvl1_restate.py.

TEST INFRASTRUCTURE: nothing in denseflow_b200/ imports it."""
import numpy as np

F = np.float32


def _planes_of(flow):
    flow = np.asarray(flow, F)
    return np.ascontiguousarray(flow[..., 0]), np.ascontiguousarray(flow[..., 1])


def farn_start(init, params=None):
    """(fx, fy) of the coarsest Farneback level from the initial flow `init` ([H,W,2] float32): orc_resize_linear to that
    level's size, times float(pyr_scale^k)"""
    from oracle import pyoracle
    L = pyoracle.lib()
    p = params or pyoracle.farn_params()
    h, w = init.shape[:2]
    levels = pyoracle.farn_levels(w, h, p)
    W, H = levels[0][:2]
    scale = 1.0
    for _ in range(len(levels) - 1):
        scale *= p.pyr_scale
    rfx, rfy = F(1.0 / (W / w)), F(1.0 / (H / h))
    fx, fy = np.empty((H, W), F), np.empty((H, W), F)
    ix, iy = _planes_of(init)
    L.orc_resize_linear(ix, w, h, fx, W, H, rfx, rfy, p.resize_convention)
    L.orc_resize_linear(iy, w, h, fy, W, H, rfx, rfy, p.resize_convention)
    return (fx * F(scale)).astype(F), (fy * F(scale)).astype(F)


def farn_calc(a, b, init=None, params=None):
    """orc_farn_calc from the C building blocks, the coarsest level starting from `init` ([H,W,2] float32, None = zero)"""
    from oracle import pyoracle
    L = pyoracle.lib()
    p = params or pyoracle.farn_params()
    a = np.ascontiguousarray(a, np.uint8)
    b = np.ascontiguousarray(b, np.uint8)
    h, w = a.shape
    levels = pyoracle.farn_levels(w, h, p)
    frames = [a.astype(F), b.astype(F)]
    fx = fy = None
    for l, (W, H, smooth, sigma) in enumerate(levels):
        if l == 0:
            fx, fy = np.zeros((H, W), F), np.zeros((H, W), F)
            if init is not None:
                fx, fy = farn_start(init, p)
        else:
            pw, ph = fx.shape[1], fx.shape[0]
            rfx, rfy = F(1.0 / (W / pw)), F(1.0 / (H / ph))
            nx, ny = np.empty((H, W), F), np.empty((H, W), F)
            L.orc_resize_linear(np.ascontiguousarray(fx), pw, ph, nx, W, H, rfx, rfy, p.resize_convention)
            L.orc_resize_linear(np.ascontiguousarray(fy), pw, ph, ny, W, H, rfx, rfy, p.resize_convention)
            mul = F(1.0 / p.pyr_scale)
            fx, fy = (nx * mul).astype(F), (ny * mul).astype(F)
        R = []
        for fr in frames:
            blurred, img = np.empty((h, w), F), np.empty((H, W), F)
            L.orc_farn_gaussian_blur(fr, w, h, smooth, sigma, blurred)
            L.orc_resize_linear(blurred, w, h, img, W, H, F(1.0 / (W / w)), F(1.0 / (H / h)), p.resize_convention)
            r = np.empty(5 * H * W, F)
            L.orc_farn_poly_exp(img, W, H, p.poly_n, p.poly_sigma, r)
            R.append(r)
        Mx, buf = np.empty(5 * H * W, F), np.empty(5 * H * W, F)
        fx, fy = np.ascontiguousarray(fx), np.ascontiguousarray(fy)
        L.orc_farn_update_matrices(fx, fy, R[0], R[1], W, H, Mx)
        for it in range(p.num_iters):
            L.orc_farn_box_filter5(Mx, W, H, p.win_size, buf)
            L.orc_farn_update_flow(buf, W, H, fx, fy)
            if it < p.num_iters - 1:
                L.orc_farn_update_matrices(fx, fy, R[0], R[1], W, H, Mx)
    return np.stack([fx, fy], -1)
