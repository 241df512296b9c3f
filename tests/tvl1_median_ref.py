"""The optional median filtering of the TV-L1 flow (`median_filtering`, `median_interval`; DESIGN §4.3) restated for the
tests, twice, with no median code shared between the two:

* `median_blur` (the contract's M_k: the element of rank (k*k - 1) / 2 of the replicate-padded k x k window, ascending, -0
  below +0, taken from integer keys in that total order) and `tvl1_calc`: the control flow of orc_tvl1_calc_ex
  (oracle/tvl1_oracle.c) over the C oracle's own building blocks, with the median inserted before every iteration n of a
  warp with n % median_interval == 0.  With the median off it is the C oracle, bit for bit (the CPU tests check that).
* `median_blur_by_value` (a partition by value, then the sign of a zero result from the count of elements below +0) and
  `numpy_calc`: oracle/tvl1_numpy.py's independent restatement of the same loop over its own building blocks.

TEST INFRASTRUCTURE: nothing in denseflow_b200/ imports it."""
import sys

import numpy as np

F = np.float32
DBL_MAX = sys.float_info.max


def _windows(u, k):
    """[H, W, k*k]: every pixel's replicate-padded window, row by row"""
    h, w = u.shape
    pad = np.pad(np.asarray(u, F), k // 2, mode="edge")
    return np.lib.stride_tricks.sliding_window_view(pad, (k, k)).reshape(h, w, k * k)


def _check_k(k):
    if k not in (3, 5):
        raise ValueError("median window must be 3 or 5, got %r" % (k,))


def median_blur(u, k):
    """M_k from keys: a float's bits as a signed integer, negatives' magnitude bits flipped (ascending, -0 below +0)"""
    _check_k(k)
    b = _windows(u, k).view(np.int32)
    keys = b ^ ((b >> 31) & 0x7fffffff)
    m = np.partition(keys, (k * k - 1) // 2, axis=-1)[..., (k * k - 1) // 2]
    return np.ascontiguousarray((m ^ ((m >> 31) & 0x7fffffff)).view(F))


def median_blur_by_value(u, k):
    """M_k by value; a zero result is -0 exactly when more than (k*k - 1) / 2 window elements lie below +0"""
    _check_k(k)
    win = _windows(u, k)
    m = (k * k - 1) // 2
    out = np.partition(win, m, axis=-1)[..., m].astype(F)
    below = ((win < 0) | ((win == 0) & np.signbit(win))).sum(-1)
    zero = out == 0
    out[zero] = np.where(below[zero] > m, F(-0.0), F(0.0))
    return out


def _median_k(median_filtering, median_interval):
    if median_filtering not in (0, 1, 3, 5) or median_interval < 1:
        raise ValueError("bad median parameters %r, %r" % (median_filtering, median_interval))
    return median_filtering if median_filtering > 1 else 0


def tvl1_calc(a, b, median_filtering=0, median_interval=30, **params):
    """orc_tvl1_calc_ex with the median, from the C building blocks.  params: pyoracle.tvl1_params keywords.  Returns
    (flow [H,W,2], iteration log [nscales, warps], convergence checks [(error, scaled_eps)]), the shape of
    pyoracle.tvl1_calc(..., return_iters=True, return_errors=True)."""
    from oracle import pyoracle
    mk = _median_k(median_filtering, median_interval)
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
    l_t, taut, theta = F(p.lambda_ * p.theta), F(p.tau / p.theta), F(p.theta)
    log = np.zeros((p.nscales, p.warps), np.int32)
    errs = []
    u1 = u2 = None
    for s in range(len(lv) - 1, -1, -1):
        W, H = lv[s]
        if u1 is None:
            u1, u2 = np.zeros((H, W), F), np.zeros((H, W), F)
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
                    u1, u2 = median_blur(u1, mk), median_blur(u2, mk)
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


def numpy_calc(I0u8, I1u8, tau=0.25, lam=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300, scale_step=0.8,
               median_filtering=0, median_interval=30):
    """oracle/tvl1_numpy.calc's loop with the median (median_blur_by_value) inserted.  Returns (flow, iteration log)."""
    from oracle import tvl1_numpy as N
    mk = _median_k(median_filtering, median_interval)
    I0s, I1s = [I0u8.astype(F)], [I1u8.astype(F)]
    finv = F(1.0 / scale_step)
    for s in range(1, nscales):
        ph, pw = I0s[-1].shape
        nw, nh = int(np.rint(pw * scale_step)), int(np.rint(ph * scale_step))
        if nw < 16 or nh < 16:
            break
        I0s.append(N.resize_cuda(I0s[-1], nw, nh, finv, finv))
        I1s.append(N.resize_cuda(I1s[-1], nw, nh, finv, finv))
    l_t, taut = F(lam * theta), F(tau / theta)
    u1 = np.zeros_like(I0s[-1])
    u2 = np.zeros_like(I0s[-1])
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
                    u1, u2 = median_blur_by_value(u1, mk), median_blur_by_value(u2, mk)
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
