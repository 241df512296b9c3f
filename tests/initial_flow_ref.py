"""`use_initial_flow` (DESIGN §1) restated for the tests.  The oracles' own entry points stay as they are; these restate them
with an initial flow, over their exported building blocks:

* `tvl1_init_pyramid` / `tvl1_calc`: the control flow of orc_tvl1_calc_ex (oracle/tvl1_oracle.c) over the C oracle's
  building blocks (as tests/tvl1_median_ref.py does, median included), with the coarsest level starting from the initial
  flow's pyramid: level 0 the field as given, level s orc_resize_linear of level s - 1 with the frame pyramid's factors
  float(1 / scale_step), then one rounded multiply by float(scale_step).
* `numpy_init_pyramid` / `numpy_calc`: the same over oracle/tvl1_numpy.py's independently written building blocks, with
  its own level sizes.
* `farn_calc`: orc_farn_calc's level loop over the C Farneback building blocks, with the coarsest level starting from
  orc_resize_linear(initial flow) to its size (explicit size, the oracle's resize convention) times float(pyr_scale^k).

With a zero initial flow each is its oracle's cold start bit for bit (tests/test_initial_flow_cpu.py checks that).

TEST INFRASTRUCTURE: nothing in denseflow_b200/ imports it."""
import sys

import numpy as np

import tvl1_median_ref as M

F = np.float32
DBL_MAX = sys.float_info.max


def _planes_of(flow):
    flow = np.asarray(flow, F)
    return np.ascontiguousarray(flow[..., 0]), np.ascontiguousarray(flow[..., 1])


def tvl1_init_pyramid(flow, lv, scale_step):
    """([u1 per level], [u2 per level]) of the initial flow [H,W,2] over the level sizes lv [(w, h), ...], C building blocks"""
    from oracle import pyoracle
    L = pyoracle.lib()
    u1, u2 = _planes_of(flow)
    p1, p2 = [u1], [u2]
    finv, mul = F(1.0 / scale_step), F(scale_step)
    for s in range(1, len(lv)):
        for pyr in (p1, p2):
            dst = np.empty((lv[s][1], lv[s][0]), F)
            L.orc_resize_linear(pyr[-1], lv[s - 1][0], lv[s - 1][1], dst, lv[s][0], lv[s][1], finv, finv, pyoracle.RESIZE_CUDA)
            pyr.append(np.ascontiguousarray(dst * mul, F))
    return p1, p2


def tvl1_calc(a, b, init=None, median_filtering=0, median_interval=30, **params):
    """orc_tvl1_calc_ex from the C building blocks, starting from `init` ([H,W,2] float32, None = zero).  params:
    pyoracle.tvl1_params keywords.  Returns (flow [H,W,2], iteration log [nscales, warps], convergence checks
    [(error, scaled_eps)]), the shape of pyoracle.tvl1_calc(..., return_iters=True, return_errors=True)."""
    from oracle import pyoracle
    mk = M._median_k(median_filtering, median_interval)
    L = pyoracle.lib()
    p = pyoracle.tvl1_params(**params)
    a = np.ascontiguousarray(a, np.uint8)
    b = np.ascontiguousarray(b, np.uint8)
    h, w = a.shape
    lv = pyoracle.tvl1_level_sizes(w, h, p)
    I0s, I1s = [a.astype(F)], [b.astype(F)]
    finv = F(1.0 / p.scale_step)
    for s in range(1, len(lv)):
        for pyr in (I0s, I1s):
            dst = np.empty((lv[s][1], lv[s][0]), F)
            L.orc_resize_linear(pyr[-1], lv[s - 1][0], lv[s - 1][1], dst, lv[s][0], lv[s][1], finv, finv, pyoracle.RESIZE_CUDA)
            pyr.append(dst)
    if init is None:
        u1, u2 = np.zeros((lv[-1][1], lv[-1][0]), F), np.zeros((lv[-1][1], lv[-1][0]), F)
    else:
        p1, p2 = tvl1_init_pyramid(init, lv, p.scale_step)
        u1, u2 = p1[-1], p2[-1]
    l_t, taut, theta = F(p.lambda_ * p.theta), F(p.tau / p.theta), F(p.theta)
    log = np.zeros((p.nscales, p.warps), np.int32)
    errs = []
    for s in range(len(lv) - 1, -1, -1):
        W, H = lv[s]
        I1x, I1y = np.empty((H, W), F), np.empty((H, W), F)
        L.orc_centered_gradient(I1s[s], W, H, I1x, I1y)
        pd = [np.zeros((H, W), F) for _ in range(4)]
        scaled_eps = p.epsilon * p.epsilon * float(W * H)
        for wi in range(p.warps):
            warped = [np.empty((H, W), F) for _ in range(5)]  # I1w, I1wx, I1wy, grad, rho_c
            L.orc_tvl1_warp_backward(I0s[s], I1s[s], I1x, I1y, u1, u2, W, H, *warped)
            error, prev, n = DBL_MAX, 0.0, 0
            while error > scaled_eps and n < p.iterations:
                if mk and n % median_interval == 0:
                    u1, u2 = M.median_blur(u1, mk), M.median_blur(u2, mk)
                calc = p.epsilon > 0 and (n & 1) and prev < scaled_eps
                e = L.orc_tvl1_estimate_u(*warped[1:], *pd, u1, u2, W, H, l_t, theta, int(bool(calc)))
                if calc:
                    error = prev = e
                    errs.append((e, scaled_eps))
                else:
                    error = DBL_MAX
                    prev -= scaled_eps
                L.orc_tvl1_estimate_dual(u1, u2, *pd, W, H, taut)
                n += 1
            log[s, wi] = n
        if s > 0:
            tw, th = lv[s - 1]
            ufx, ufy = F(1.0 / (tw / W)), F(1.0 / (th / H))
            mul = F(1.0 / p.scale_step)
            up = []
            for u in (u1, u2):
                dst = np.empty((th, tw), F)
                L.orc_resize_linear(u, W, H, dst, tw, th, ufx, ufy, pyoracle.RESIZE_CUDA)
                up.append(np.ascontiguousarray(dst * mul, F))
            u1, u2 = up
    return np.stack([u1, u2], -1), log, np.array(errs, np.float64).reshape(-1, 2)


def _numpy_levels(h, w, nscales, scale_step):
    sizes = [(w, h)]
    for _ in range(1, nscales):
        pw, ph = sizes[-1]
        nw, nh = int(np.rint(pw * scale_step)), int(np.rint(ph * scale_step))
        if nw < 16 or nh < 16:
            break
        sizes.append((nw, nh))
    return sizes


def numpy_init_pyramid(flow, nscales, scale_step):
    """tvl1_init_pyramid over oracle/tvl1_numpy.py's resize and its own level sizes"""
    from oracle import tvl1_numpy as N
    u1, u2 = _planes_of(flow)
    sizes = _numpy_levels(u1.shape[0], u1.shape[1], nscales, scale_step)
    finv = F(1.0 / scale_step)
    p1, p2 = [u1], [u2]
    for nw, nh in sizes[1:]:
        p1.append((N.resize_cuda(p1[-1], nw, nh, finv, finv) * F(scale_step)).astype(F))
        p2.append((N.resize_cuda(p2[-1], nw, nh, finv, finv) * F(scale_step)).astype(F))
    return p1, p2


def numpy_calc(I0u8, I1u8, init=None, tau=0.25, lam=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300,
               scale_step=0.8, median_filtering=0, median_interval=30):
    """oracle/tvl1_numpy.calc's loop starting from `init` (None = zero), median as tests/tvl1_median_ref.numpy_calc.
    Returns (flow, iteration log)."""
    from oracle import tvl1_numpy as N
    mk = M._median_k(median_filtering, median_interval)
    I0s, I1s = [I0u8.astype(F)], [I1u8.astype(F)]
    finv = F(1.0 / scale_step)
    for nw, nh in _numpy_levels(I0u8.shape[0], I0u8.shape[1], nscales, scale_step)[1:]:
        I0s.append(N.resize_cuda(I0s[-1], nw, nh, finv, finv))
        I1s.append(N.resize_cuda(I1s[-1], nw, nh, finv, finv))
    if init is None:
        u1, u2 = np.zeros_like(I0s[-1]), np.zeros_like(I0s[-1])
    else:
        p1, p2 = numpy_init_pyramid(init, nscales, scale_step)
        u1, u2 = p1[len(I0s) - 1], p2[len(I0s) - 1]
    l_t, taut = F(lam * theta), F(tau / theta)
    log = np.zeros((nscales, warps), np.int32)
    for s in range(len(I0s) - 1, -1, -1):
        I0, I1 = I0s[s], I1s[s]
        h, w = I0.shape
        I1x, I1y = N.gradient(I1)
        p11, p12, p21, p22 = (np.zeros_like(I0) for _ in range(4))
        scaled_eps = epsilon * epsilon * (w * h)
        for wi in range(warps):
            ix, iy, grad, rho_c = N.warp(I0, I1, I1x, I1y, u1, u2)
            error, prev, it = np.finfo(np.float64).max, 0.0, 0
            while error > scaled_eps and it < iterations:
                if mk and it % median_interval == 0:
                    u1, u2 = M.median_blur_by_value(u1, mk), M.median_blur_by_value(u2, mk)
                calc_err = epsilon > 0 and (it & 1) and prev < scaled_eps
                u1, u2, e = N.estimate_u(ix, iy, grad, rho_c, p11, p12, p21, p22, u1, u2, l_t, F(theta))
                if calc_err:
                    error = prev = e
                else:
                    error = np.finfo(np.float64).max
                    prev -= scaled_eps
                p11, p12, p21, p22 = N.estimate_dual(u1, u2, p11, p12, p21, p22, taut)
                it += 1
            log[s, wi] = it
        if s > 0:
            th, tw = I0s[s - 1].shape
            ufx, ufy = F(1.0 / (tw / w)), F(1.0 / (th / h))
            u1 = (N.resize_cuda(u1, tw, th, ufx, ufy) * F(1.0 / scale_step)).astype(F)
            u2 = (N.resize_cuda(u2, tw, th, ufx, ufy) * F(1.0 / scale_step)).astype(F)
    return np.stack([u1, u2], -1), log


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
