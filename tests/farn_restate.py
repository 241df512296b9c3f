"""Farneback with the options the oracle does not have, restated for the tests: a warm start (`use_initial_flow`, DESIGN
§1), the Gaussian window (`gaussian_window`, OPTFLOW_FARNEBACK_GAUSSIAN) and fast pyramids (`fast_pyramids`,
fastPyramids), the last two per SURVEY Appendix B.7.  The oracle's own entry point stays as it is.

`farn_calc` is orc_farn_calc's level loop over the C oracle's building blocks (orc_farn_update_matrices,
orc_farn_update_flow, orc_farn_poly_exp, orc_resize_linear, and for B.1 level images orc_farn_gaussian_blur).  With no
initial flow or a zero one and both options off it is orc_farn_calc bit for bit (tests/test_initial_flow_cpu.py and
tests/test_farn_window_cpu.py check that).  What each option adds to the loop:

* Warm start: the coarsest level starts from `farn_start`: orc_resize_linear(initial flow) to that level's size (explicit
  size, the oracle's resize convention) times float(pyr_scale^k).
* Gaussian window: the 13x13 Gaussian window (`gauss_window5`) in numpy fp32 takes the place of the box mean.
* Fast pyramids: the pyrDown chain (`pyr_down`) in numpy fp32 builds the level images, at its own level sizes
  (`level_sizes`).

Every fp32 step of the window and the pyrDown chain is one numpy elementwise operation on float32 arrays (one rounding
each, no fused multiply-add), in the contract's order, so the strict build can be compared with it bit for bit.  The
TV-L1 options are restated in tests/tvl1_restate.py.

TEST INFRASTRUCTURE: nothing in denseflow_b200/ imports it."""
import math

import numpy as np

from farn_ref64 import reflect101

F = np.float32
WIN = 13
PYR_K = [F(0.0625), F(0.25), F(0.375), F(0.25), F(0.0625)]


def gauss_weights(ksize=WIN):
    """getGaussianKernel(ksize, (float)(ksize / 2) * 0.3f, CV_32F), centre and right half, computed as the engine computes
    it: the fp32 sigma widened to double, exp / sum / scale in double, then cast to fp32"""
    half = ksize // 2
    sigma = float(F(half) * F(0.3))
    scale2x = -0.5 / (sigma * sigma)
    t = [math.exp(scale2x * (i - (ksize - 1) * 0.5) ** 2) for i in range(ksize)]
    s = 0.0
    for v in t:
        s += v
    s = 1.0 / s
    return np.array([t[half + i] * s for i in range(half + 1)], F)


def gauss_window5(M):
    """B.7: the five planes of M ([5, h, w] float32) each filtered by the separable 13x13 Gaussian window, index-clamped
    rows and columns, vertical pass first; each pass is acc = s(0) g0, then acc += (s(-j) + s(+j)) gj for j = 1..6"""
    g = gauss_weights()
    half = len(g) - 1
    M = np.asarray(M, F)
    h, w = M.shape[1:]
    yi, xi = np.arange(h), np.arange(w)
    out = np.empty_like(M)
    for k in range(5):
        P = M[k]
        acc = P * g[0]
        for j in range(1, half + 1):
            acc = acc + (P[np.maximum(yi - j, 0)] + P[np.minimum(yi + j, h - 1)]) * g[j]
        v = acc
        acc = v * g[0]
        for j in range(1, half + 1):
            acc = acc + (v[:, np.maximum(xi - j, 0)] + v[:, np.minimum(xi + j, w - 1)]) * g[j]
        out[k] = acc
    return out


def pyr_down(img):
    """cv::cuda::pyrDown, BORDER_REFLECT_101: output ((w + 1) / 2, (h + 1) / 2); the vertical pass then the horizontal pass
    each sum 0.0625 s(-2) + 0.25 s(-1) + 0.375 s(0) + 0.25 s(+1) + 0.0625 s(+2) left to right in fp32, at source row / column
    2y / 2x"""
    img = np.asarray(img, F)
    h, w = img.shape
    dh, dw = (h + 1) // 2, (w + 1) // 2
    ry, cx = 2 * np.arange(dh), 2 * np.arange(dw)
    v = img[reflect101(ry - 2, h)] * PYR_K[0]
    for d in range(1, 5):
        v = v + img[reflect101(ry + d - 2, h)] * PYR_K[d]
    out = v[:, reflect101(cx - 2, w)] * PYR_K[0]
    for e in range(1, 5):
        out = out + v[:, reflect101(cx + e - 2, w)] * PYR_K[e]
    return out


def level_sizes(w, h, params=None, fast_pyramids=0):
    """the level sizes (w, h) in processing order (coarsest first): B.1's count always; B.1's cvRound sizes, or with
    fast_pyramids the pyrDown chain's ((w + 1) / 2, (h + 1) / 2) per level"""
    from oracle import pyoracle
    levels = pyoracle.farn_levels(w, h, params or pyoracle.farn_params())
    if not fast_pyramids:
        return [lv[:2] for lv in levels]
    sizes = [(w, h)]
    for _ in range(len(levels) - 1):
        pw, ph = sizes[-1]
        sizes.append(((pw + 1) // 2, (ph + 1) // 2))
    return sizes[::-1]


def _resize(L, src, W, H, conv):
    h, w = src.shape
    out = np.empty((H, W), F)
    L.orc_resize_linear(np.ascontiguousarray(src, F), w, h, out, W, H, F(1.0 / (W / w)), F(1.0 / (H / h)), conv)
    return out


def farn_start(init, params=None, *, fast_pyramids=0):
    """(fx, fy) of the coarsest level from the initial flow `init` ([H,W,2] float32): orc_resize_linear to the size that
    level has in the driver (level_sizes(...)[0]), times float(pyr_scale^k)"""
    from oracle import pyoracle
    L = pyoracle.lib()
    p = params or pyoracle.farn_params()
    init = np.asarray(init, F)
    h, w = init.shape[:2]
    sizes = level_sizes(w, h, p, fast_pyramids)
    W, H = sizes[0]
    scale = 1.0
    for _ in range(len(sizes) - 1):
        scale *= p.pyr_scale
    return tuple((_resize(L, init[..., c], W, H, p.resize_convention) * F(scale)).astype(F) for c in (0, 1))


def farn_calc(a, b, *, init=None, params=None, gaussian_window=0, fast_pyramids=0):
    """orc_farn_calc with the two B.7 options, the coarsest level starting from farn_start(init) ([H,W,2] float32, None =
    zero)"""
    from oracle import pyoracle
    L = pyoracle.lib()
    p = params or pyoracle.farn_params()
    a = np.ascontiguousarray(a, np.uint8)
    b = np.ascontiguousarray(b, np.uint8)
    h, w = a.shape
    levels = pyoracle.farn_levels(w, h, p)
    sizes = level_sizes(w, h, p, fast_pyramids)
    n = len(levels)
    frames = [a.astype(F), b.astype(F)]
    if fast_pyramids:  # level k = pyrDown(level k - 1), level 0 the unblurred frame; stored coarsest first
        pyrs = []
        for fr in frames:
            chain = [fr]
            for _ in range(n - 1):
                chain.append(pyr_down(chain[-1]))
            pyrs.append(chain[::-1])
    fx = fy = None
    for l, (W, H) in enumerate(sizes):
        if l == 0:
            fx, fy = np.zeros((H, W), F), np.zeros((H, W), F)
            if init is not None:
                fx, fy = farn_start(init, p, fast_pyramids=fast_pyramids)
        else:
            mul = F(1.0 / p.pyr_scale)
            fx = (_resize(L, fx, W, H, p.resize_convention) * mul).astype(F)
            fy = (_resize(L, fy, W, H, p.resize_convention) * mul).astype(F)
        R = []
        for i, fr in enumerate(frames):
            if fast_pyramids:
                img = np.ascontiguousarray(pyrs[i][l])
            else:
                smooth, sigma = levels[l][2:]
                blurred = np.empty((h, w), F)
                L.orc_farn_gaussian_blur(fr, w, h, smooth, sigma, blurred)
                img = _resize(L, blurred, W, H, p.resize_convention)
            r = np.empty(5 * H * W, F)
            L.orc_farn_poly_exp(img, W, H, p.poly_n, p.poly_sigma, r)
            R.append(r)
        Mx, buf = np.empty(5 * H * W, F), np.empty(5 * H * W, F)
        fx, fy = np.ascontiguousarray(fx), np.ascontiguousarray(fy)
        L.orc_farn_update_matrices(fx, fy, R[0], R[1], W, H, Mx)
        for it in range(p.num_iters):
            if gaussian_window:
                buf = np.ascontiguousarray(gauss_window5(Mx.reshape(5, H, W)).reshape(-1))
            else:
                L.orc_farn_box_filter5(Mx, W, H, p.win_size, buf)
            L.orc_farn_update_flow(buf, W, H, fx, fy)
            if it < p.num_iters - 1:
                L.orc_farn_update_matrices(fx, fy, R[0], R[1], W, H, Mx)
    return np.stack([fx, fy], -1)
