"""TV-L1 with the options the oracles do not have, restated for the tests: the median filtering of the flow
(`median_filtering`, `median_interval`; DESIGN §4.3), a warm start (`use_initial_flow`, DESIGN §1) and the illumination
term (`gamma`; SURVEY.md A.8).  Two restatements, each with every option, sharing no median, divergence or dual code:

* `tvl1_calc`: the control flow of orc_tvl1_calc_ex (oracle/tvl1_oracle.c) over the C oracle's own building blocks.  With
  the median off, no initial flow and gamma = 0 it runs the C oracle's own steps, so it is the C oracle bit for bit (the CPU
  tests check that).
* `numpy_calc`: oracle/tvl1_numpy.py's independent restatement of the same loop over its own building blocks and its own
  level sizes.

What each option adds to the loop:

* Median: M_k is the element of rank (k*k - 1) / 2 of the replicate-padded k x k window, ascending, -0 below +0.
  `median_blur` (C side) takes it from integer keys in that total order; `median_blur_by_value` (numpy side) partitions by
  value and then takes the sign of a zero result from the count of elements below +0.  The median of u1 and u2 runs before
  every iteration n of a warp with n % median_interval == 0.
* Warm start: the coarsest level starts from the initial flow's pyramid instead of zero (it is not zeroed): level 0 the
  field as given, level s orc_resize_linear of level s - 1 with the frame pyramid's factors float(1 / scale_step), then one
  rounded multiply by float(scale_step) (`tvl1_init_pyramid`, `numpy_init_pyramid`).
* Gamma > 0: the primal step `estimate_u_gamma` (the oracle's estimate_u with gamma * u3 in rho, d3 and u3, written after
  the C source), the dual step `estimate_dual_gamma` (orc_tvl1_estimate_dual on u1, u2 and again on u3 alone, so the dual
  step on u3 runs through the C oracle's dual step) and the u3 resize between scales (`resize_u3`: orc_resize_linear with the
  flow's factors, no 1 / scale_step).  u3 starts at 0 on the coarsest level, also when warm-started; p31 and p32 are zeroed
  at every scale as p11..p22 are.  The numpy side writes the same steps over its own divergence, with |grad u3| from
  np.hypot as it takes |grad u1|.

TEST INFRASTRUCTURE: nothing in denseflow_b200/ imports it."""
import sys

import numpy as np

F = np.float32
DBL_MAX = sys.float_info.max
FLT_EPS = np.finfo(F).eps


# ---- median ----------------------------------------------------------------------------------------------------------------
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


# ---- warm start ------------------------------------------------------------------------------------------------------------
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


# ---- gamma ---------------------------------------------------------------------------------------------------------------
def _check_gamma(gamma):
    if not (np.isfinite(gamma) and gamma >= 0):
        raise ValueError("bad gamma %r" % (gamma,))


def _div_c(pa, pb):
    """the C oracle's divergence(): (pa - pa_left) + (pb - pb_up) inside, (pa + pb) - pb_up on column 0, (pa - pa_left) + pb
    on row 0, pa + pb in the corner"""
    out = np.empty_like(pa)
    out[1:, 1:] = (pa[1:, 1:] - pa[1:, :-1]) + (pb[1:, 1:] - pb[:-1, 1:])
    out[1:, 0] = (pa[1:, 0] + pb[1:, 0]) - pb[:-1, 0]
    out[0, 1:] = (pa[0, 1:] - pa[0, :-1]) + pb[0, 1:]
    out[0, 0] = pa[0, 0] + pb[0, 0]
    return out


def estimate_u_gamma(ix, iy, grad, rho_c, p11, p12, p21, p22, p31, p32, u1, u2, u3, l_t, theta, gamma):
    """The primal step with u3, every operation rounded to fp32 in the C source's order.  Returns (u1', u2', u3', the
    convergence error sum((du1)^2 + (du2)^2) in double)."""
    l_t, theta, gamma = F(l_t), F(theta), F(gamma)
    rho = rho_c + ((ix * u1 + iy * u2) + gamma * u3)
    thr = l_t * grad
    with np.errstate(divide="ignore", invalid="ignore"):
        fi = -rho / grad
    f = np.where(rho < -thr, l_t, np.where(rho > thr, -l_t, np.where(grad > FLT_EPS, fi, F(0)))).astype(F)
    n1 = (u1 + f * ix) + theta * _div_c(p11, p12)
    n2 = (u2 + f * iy) + theta * _div_c(p21, p22)
    n3 = (u3 + f * gamma) + theta * _div_c(p31, p32)
    e = ((u1 - n1) * (u1 - n1) + (u2 - n2) * (u2 - n2)).astype(np.float64).sum()
    return n1.astype(F), n2.astype(F), n3.astype(F), float(e)


def estimate_dual_gamma(u1, u2, u3, p, taut):
    """p = [p11, p12, p21, p22, p31, p32], updated in place by the C oracle's dual step: on (u1, u2) as it is, and on u3 through
    its first field (the second pair of planes it writes is scratch)"""
    from oracle import pyoracle
    L = pyoracle.lib()
    h, w = u1.shape
    L.orc_tvl1_estimate_dual(u1, u2, *p[:4], w, h, F(taut))
    scratch = [np.zeros_like(u3), np.zeros_like(u3)]
    L.orc_tvl1_estimate_dual(u3, u3, p[4], p[5], *scratch, w, h, F(taut))


def resize_u3(u3, tw, th):
    """u3 to the next finer level: orc_resize_linear with the flow's factors, not multiplied"""
    from oracle import pyoracle
    h, w = u3.shape
    dst = np.empty((th, tw), F)
    pyoracle.lib().orc_resize_linear(np.ascontiguousarray(u3, F), w, h, dst, tw, th, F(1.0 / (tw / w)), F(1.0 / (th / h)),
                                     pyoracle.RESIZE_CUDA)
    return dst


def _numpy_estimate_u(N, ix, iy, grad, rho_c, p, u1, u2, u3, l_t, theta, gamma):
    rho = (rho_c + ((ix * u1 + iy * u2).astype(F) + (F(gamma) * u3).astype(F)).astype(F)).astype(F)
    thr = (F(l_t) * grad).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        fi = (-rho / grad).astype(F)
    f = np.zeros_like(u1)
    f = np.where(grad > np.finfo(F).eps, fi, f)
    f = np.where(rho > thr, -F(l_t), f)
    f = np.where(rho < -thr, F(l_t), f).astype(F)
    outs = []
    for u, d, (pa, pb) in ((u1, f * ix, p[0:2]), (u2, f * iy, p[2:4]), (u3, f * F(gamma), p[4:6])):
        outs.append(((u + d.astype(F)).astype(F) + (F(theta) * N.divergence(pa, pb)).astype(F)).astype(F))
    n1, n2, n3 = outs
    diff = (((u1 - n1) * (u1 - n1)).astype(F) + ((u2 - n2) * (u2 - n2)).astype(F)).astype(F)
    return n1, n2, n3, float(diff.astype(np.float64).sum())


def _numpy_dual_u3(u3, p31, p32, taut):
    ux = (np.concatenate([u3[:, 1:], u3[:, -1:]], 1) - u3).astype(F)
    uy = (np.concatenate([u3[1:], u3[-1:]], 0) - u3).astype(F)
    ng = (F(1) + F(taut) * np.hypot(ux.astype(np.float64), uy.astype(np.float64)).astype(F)).astype(F)
    return ((p31 + F(taut) * ux).astype(F) / ng).astype(F), ((p32 + F(taut) * uy).astype(F) / ng).astype(F)


# ---- the two pyramid drivers -----------------------------------------------------------------------------------------------
def tvl1_calc(a, b, *, init=None, median_filtering=0, median_interval=30, gamma=0.0, return_u3=False, **params):
    """orc_tvl1_calc_ex from the C building blocks, starting from `init` ([H,W,2] float32, None = zero).  params:
    pyoracle.tvl1_params keywords.  Returns (flow [H,W,2], iteration log [nscales, warps], convergence checks
    [(error, scaled_eps)]), the shape of pyoracle.tvl1_calc(..., return_iters=True, return_errors=True), and, with
    return_u3, the level-0 u3 last."""
    from oracle import pyoracle
    _check_gamma(gamma)
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
    if init is None:
        u1, u2 = np.zeros((lv[-1][1], lv[-1][0]), F), np.zeros((lv[-1][1], lv[-1][0]), F)
    else:
        p1, p2 = tvl1_init_pyramid(init, lv, p.scale_step)
        u1, u2 = p1[-1], p2[-1]
    u3 = np.zeros((lv[-1][1], lv[-1][0]), F)
    l_t, taut, theta = F(p.lambda_ * p.theta), F(p.tau / p.theta), F(p.theta)
    log = np.zeros((p.nscales, p.warps), np.int32)
    errs = []
    for s in range(len(lv) - 1, -1, -1):
        W, H = lv[s]
        I1x, I1y = np.empty((H, W), F), np.empty((H, W), F)
        L.orc_centered_gradient(I1s[s], W, H, I1x, I1y)
        pd = [np.zeros((H, W), F) for _ in range(6)]
        scaled_eps = p.epsilon * p.epsilon * float(W * H)
        for wi in range(p.warps):
            warped = [np.empty((H, W), F) for _ in range(5)]  # I1w, I1wx, I1wy, grad, rho_c
            L.orc_tvl1_warp_backward(I0s[s], I1s[s], I1x, I1y, u1, u2, W, H, *warped)
            error, prev, n = DBL_MAX, 0.0, 0
            while error > scaled_eps and n < p.iterations:
                if mk and n % median_interval == 0:
                    u1, u2 = median_blur(u1, mk), median_blur(u2, mk)
                calc = p.epsilon > 0 and (n & 1) and prev < scaled_eps
                if gamma > 0:
                    u1, u2, u3, e = estimate_u_gamma(*warped[1:], *pd, u1, u2, u3, l_t, theta, gamma)
                else:
                    e = L.orc_tvl1_estimate_u(*warped[1:], *pd[:4], u1, u2, W, H, l_t, theta, int(bool(calc)))
                if calc:
                    error = prev = e
                    errs.append((e, scaled_eps))
                else:
                    error = DBL_MAX
                    prev -= scaled_eps
                if gamma > 0:
                    estimate_dual_gamma(u1, u2, u3, pd, taut)
                else:
                    L.orc_tvl1_estimate_dual(u1, u2, *pd[:4], W, H, taut)
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
            u3 = resize_u3(u3, tw, th)
    out = (np.stack([u1, u2], -1), log, np.array(errs, np.float64).reshape(-1, 2))
    return out + (u3,) if return_u3 else out


def numpy_calc(I0u8, I1u8, *, init=None, median_filtering=0, median_interval=30, gamma=0.0, tau=0.25, lam=0.15, theta=0.3,
               nscales=5, warps=5, epsilon=0.01, iterations=300, scale_step=0.8, return_u3=False):
    """oracle/tvl1_numpy.calc's loop, starting from `init` (None = zero).  Returns (flow, iteration log) and, with return_u3,
    the level-0 u3."""
    from oracle import tvl1_numpy as N
    _check_gamma(gamma)
    mk = _median_k(median_filtering, median_interval)
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
    u3 = np.zeros_like(I0s[-1])
    l_t, taut = F(lam * theta), F(tau / theta)
    log = np.zeros((nscales, warps), np.int32)
    for s in range(len(I0s) - 1, -1, -1):
        I0, I1 = I0s[s], I1s[s]
        h, w = I0.shape
        I1x, I1y = N.gradient(I1)
        p = [np.zeros_like(I0) for _ in range(6)]
        scaled_eps = epsilon * epsilon * (w * h)
        for wi in range(warps):
            ix, iy, grad, rho_c = N.warp(I0, I1, I1x, I1y, u1, u2)
            error, prev, it = np.finfo(np.float64).max, 0.0, 0
            while error > scaled_eps and it < iterations:
                if mk and it % median_interval == 0:
                    u1, u2 = median_blur_by_value(u1, mk), median_blur_by_value(u2, mk)
                calc_err = epsilon > 0 and (it & 1) and prev < scaled_eps
                if gamma > 0:
                    u1, u2, u3, e = _numpy_estimate_u(N, ix, iy, grad, rho_c, p, u1, u2, u3, l_t, theta, gamma)
                else:
                    u1, u2, e = N.estimate_u(ix, iy, grad, rho_c, *p[:4], u1, u2, l_t, F(theta))
                if calc_err:
                    error = prev = e
                else:
                    error = np.finfo(np.float64).max
                    prev -= scaled_eps
                p[:4] = N.estimate_dual(u1, u2, *p[:4], taut)
                if gamma > 0:
                    p[4:6] = _numpy_dual_u3(u3, p[4], p[5], taut)
                it += 1
            log[s, wi] = it
        if s > 0:
            th, tw = I0s[s - 1].shape
            ufx, ufy = F(1.0 / (tw / w)), F(1.0 / (th / h))
            u1 = (N.resize_cuda(u1, tw, th, ufx, ufy) * F(1.0 / scale_step)).astype(F)
            u2 = (N.resize_cuda(u2, tw, th, ufx, ufy) * F(1.0 / scale_step)).astype(F)
            u3 = N.resize_cuda(u3, tw, th, ufx, ufy)
    flow = np.stack([u1, u2], -1)
    return (flow, log, u3) if return_u3 else (flow, log)
