"""Float64 restatement of each Farneback stage, with a forward-error bound for its fp32 evaluation.

Every stage takes the same fp32 inputs as the kernel (and as the oracle's building block) and returns, per output plane, the
float64 value of the operation and a bound on |fp32 result - float64 value| derived from the operation itself:

* Sums and products are evaluated on `E` values that carry, next to the float64 value, the magnitude of the expression
  (the same expression on absolute values, subtractions turned into additions) and its rounding depth k (the largest
  number of rounded fp32 operations on a path from an input to the result).  For such a tree
  |fl(y) - y| <= gamma_k * magnitude, gamma_k = k u / (1 - k u), u = 2^-24 (Higham, Accuracy and Stability of Numerical
  Algorithms, §3.1).  Fused multiply-adds only remove roundings, so the bound holds for the default build too.
  A rounded operation on two exact inputs contributes |result| as its magnitude (it is off by one relative rounding).
* Filter weights and polynomial-expansion constants are fp32 values computed in double and cast; the engine computes them
  with its own code, so they enter as inputs one rounding away (depth 1) instead of exact.
* The 2x2 solve divides: numerator N and denominator D come with their own bounds eN, eD, then
  |N^/D^ - N/D| <= (eN + |N| eD / |D|) / (|D| - eD), and the reciprocal (rcp.approx: 2 ulp, i.e. 4u relative) and the
  final multiply (u) add their relative error on top.
* Every rounding in the subnormal range may add 2^-150 absolutely: k * 2^-150.  The float64 restatement rounds as well
  (u = 2^-53, same depth), so gamma_k uses u = 2^-24 + 2^-53.
Coordinates (x + dx, its floor and fraction, dx * rfx) are single IEEE operations on inputs, computed here in fp32 exactly
as the kernels and the oracle do, and then used as exact values.
"""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -150
C_BORDER = np.array([0.14, 0.14, 0.4472, 0.4472, 0.4472, 1.0], np.float32)


def gamma(k):
    u = U + 2.0 ** -53  # the float64 restatement rounds too, with the same rounding depth
    return k * u / (1.0 - k * u)


class E:
    """float64 value `v`, magnitude `m`, rounding depth `d` of one fp32 expression (element-wise over arrays)."""
    __slots__ = ("v", "m", "d")

    def __init__(self, v, m=None, d=0):
        self.v = np.asarray(v, np.float64)
        self.m = np.abs(self.v) if m is None else m
        self.d = d

    @staticmethod
    def lift(o):
        return o if isinstance(o, E) else E(o)

    def _op(self, o, v, m):
        if self.d == 0 and o.d == 0:
            return E(v, np.abs(v), 1)
        return E(v, m, max(self.d, o.d) + 1)

    def __add__(self, o):
        o = E.lift(o)
        return self._op(o, self.v + o.v, self.m + o.m)

    def __sub__(self, o):
        o = E.lift(o)
        return self._op(o, self.v - o.v, self.m + o.m)

    def __mul__(self, o):
        o = E.lift(o)
        return self._op(o, self.v * o.v, self.m * o.m)

    def scale2(self, c):
        """multiplication by a power of two: exact"""
        return E(self.v * c, self.m * abs(c), self.d)

    def __getitem__(self, idx):
        return E(self.v[idx], self.m[idx], self.d)

    @staticmethod
    def where(c, a, b):
        return E(np.where(c, a.v, b.v), np.where(c, a.m, b.m), max(a.d, b.d))

    def bound(self):
        return gamma(self.d) * self.m + self.d * TINY

    def out(self):
        return self.v, self.bound()


def const(x):
    """an fp32 constant the engine derives with its own code: one rounding away from this one"""
    return E(np.float32(x), d=1)


def reflect101(i, n):
    i = np.asarray(i)
    if n == 1:
        return np.zeros_like(i)
    while ((i < 0) | (i >= n)).any():
        i = np.where(i < 0, -i, np.where(i >= n, 2 * (n - 1) - i, i))
    return i


def cv_round(v):
    return int(round(v))  # half to even, like nearbyint


def levels(w, h, num_levels=5, pyr_scale=0.5):
    """B.1 level list in processing order (coarsest first): (w, h, smooth_size, sigma)"""
    cropped, scale = 0, 1.0
    while cropped < num_levels:
        scale *= pyr_scale
        if w * scale < 32 or h * scale < 32:
            break
        cropped += 1
    out = []
    for k in range(cropped, -1, -1):
        scale = pyr_scale ** k
        sigma = (1.0 / scale - 1) * 0.5
        out.append((cv_round(w * scale), cv_round(h * scale), max(cv_round(sigma * 5) | 1, 3), sigma))
    return out


def gaussian_half_kernel(ksize, sigma):
    """cv::getGaussianKernel(ksize, sigma, CV_32F), centre and right half; `exact` for the fixed dyadic tables"""
    half = ksize // 2
    tabs = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
            7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125]}
    if ksize % 2 == 1 and ksize <= 7 and sigma <= 0:
        return np.array(tabs[ksize][half:], np.float32), True
    sx = sigma if sigma > 0 else ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8
    x = np.arange(ksize) - (ksize - 1) * 0.5
    t = np.exp(-0.5 / (sx * sx) * x * x)
    return (t[half:] * (1.0 / t.sum())).astype(np.float32), False


def poly_constants(n=5, sigma=1.1):
    """B.3 constants: g, xg, xxg (k = 0..n) and ig11, ig03, ig33, ig55"""
    if sigma < 1.1920928955078125e-7:
        sigma = n * 0.3
    x = np.arange(-n, n + 1)
    g = np.exp(-x * x / (2 * sigma * sigma)).astype(np.float32)
    g = (g.astype(np.float64) * (1.0 / g.astype(np.float64).sum())).astype(np.float32)
    xf = x.astype(np.float32)
    xg = xf * g  # int * float: fp32 products, as upstream
    xxg = (xf * xf) * g
    gy, gx = np.meshgrid(g, g, indexing="ij")
    yy, xx = np.meshgrid(xf, xf, indexing="ij")
    G = np.zeros((6, 6))
    G[0, 0] = (gy * gx).astype(np.float64).sum()
    G[1, 1] = (gy * gx * xx * xx).astype(np.float64).sum()
    G[3, 3] = (gy * gx * xx * xx * xx * xx).astype(np.float64).sum()
    G[5, 5] = (gy * gx * xx * xx * yy * yy).astype(np.float64).sum()
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    iG = np.linalg.inv(G)
    ig = np.array([iG[1, 1], iG[0, 3], iG[3, 3], iG[5, 5]], np.float32)
    return g[n:], xg[n:], xxg[n:], ig


def _resize_coords(dn, sn, rf):
    """CUDA resize_linear sampling: s = d * rf in fp32, floor, the far tap clamped"""
    s = np.arange(dn, dtype=np.float32) * np.float32(rf)
    i1 = np.floor(s).astype(np.int64)
    return s, i1, np.minimum(i1, sn - 1), np.minimum(i1 + 1, sn - 1)


def _bilinear4(b, sx, x1, sy, y1):
    """out = b00 (x2-sx)(y2-sy) + b01 (sx-x1)(y2-sy) + b10 (x2-sx)(sy-y1) + b11 (sx-x1)(sy-y1), summed in that order"""
    ex2, ex1, esx = E(x1 + 1.0), E(x1 * 1.0), E(sx)
    ey2, ey1, esy = E(y1 + 1.0), E(y1 * 1.0), E(sy)
    wx = (ex2 - esx, esx - ex1)
    wy = (ey2 - esy, esy - ey1)
    out = b[0][0] * (wx[0] * wy[0])
    out = out + b[0][1] * (wx[1] * wy[0])
    out = out + b[1][0] * (wx[0] * wy[1])
    return out + b[1][1] * (wx[1] * wy[1])


def level_image(frame, lw, lh, ksize, sigma):
    """B.2: Gaussian blur (BORDER_REFLECT_101, vertical pass first) of the full-resolution frame, bilinear resize to lw x lh"""
    frame = np.asarray(frame, np.float32)
    H, W = frame.shape
    k, exact = gaussian_half_kernel(ksize, sigma)
    kw = [E(k[j]) if exact else const(k[j]) for j in range(len(k))]
    half = len(k) - 1
    rfx = np.float32(1.0 / (lw / W))
    rfy = np.float32(1.0 / (lh / H))
    sx, x1, xa, xb = _resize_coords(lw, W, rfx)
    sy, y1, ya, yb = _resize_coords(lh, H, rfy)

    def vert(rows):
        acc = E(frame[rows]) * kw[0]
        for j in range(1, half + 1):
            acc = acc + (E(frame[reflect101(rows - j, H)]) + E(frame[reflect101(rows + j, H)])) * kw[j]
        return acc

    def horz(V, cols):
        acc = V[:, cols] * kw[0]
        for j in range(1, half + 1):
            acc = acc + (V[:, reflect101(cols - j, W)] + V[:, reflect101(cols + j, W)]) * kw[j]
        return acc

    b = [[horz(V, c) for c in (xa, xb)] for V in (vert(ya), vert(yb))]
    return _bilinear4(b, sx[None, :], x1[None, :], sy[:, None], y1[:, None]).out()


def poly_exp(img, n=5, sigma=1.1):
    """B.3: polynomial expansion, index-clamped borders, vertical pass (t0, t1, t2) then horizontal: R0 .. R4"""
    img = np.asarray(img, np.float32)
    h, w = img.shape
    g, xg, xxg, ig = poly_constants(n, sigma)
    g, xg, xxg = [[const(c) for c in a] for a in (g, xg, xxg)]
    ig11, ig03, ig33, ig55 = [const(c) for c in ig]
    yi, xi = np.arange(h), np.arange(w)
    a0 = E(img) * g[0]
    a1 = a2 = None
    for k in range(1, n + 1):
        s0, s1 = E(img[np.maximum(yi - k, 0)]), E(img[np.minimum(yi + k, h - 1)])
        a0 = a0 + g[k] * (s0 + s1)
        t1, t2 = xg[k] * (s1 - s0), xxg[k] * (s0 + s1)
        a1 = t1 if a1 is None else a1 + t1  # 0 + t: exact
        a2 = t2 if a2 is None else a2 + t2
    b1, b3, b5 = g[0] * a0, g[0] * a1, g[0] * a2
    b2 = b4 = b6 = None
    for k in range(1, n + 1):
        xl, xr = np.maximum(xi - k, 0), np.minimum(xi + k, w - 1)
        s = a0[:, xr] + a0[:, xl]
        b1 = b1 + s * g[k]
        b4 = s * xxg[k] if b4 is None else b4 + s * xxg[k]
        t = (a0[:, xr] - a0[:, xl]) * xg[k]
        b2 = t if b2 is None else b2 + t
        s = a1[:, xr] + a1[:, xl]
        b3 = b3 + s * g[k]
        t = (a1[:, xr] - a1[:, xl]) * xg[k]
        b6 = t if b6 is None else b6 + t
        s = a2[:, xr] + a2[:, xl]
        b5 = b5 + s * g[k]
    R = [b3 * ig11, b2 * ig11, b1 * ig03 + b5 * ig33, b1 * ig03 + b4 * ig33, b6 * ig55]
    return [r.out() for r in R]


def _update_matrices_e(fx, fy, R0, R1):
    fx = np.asarray(fx, np.float32)
    fy = np.asarray(fy, np.float32)
    h, w = fx.shape
    yy, xx = np.mgrid[0:h, 0:w]
    px = xx.astype(np.float32) + fx  # fp32, as the kernel
    py = yy.astype(np.float32) + fy
    x1 = np.floor(px).astype(np.int64)
    y1 = np.floor(py).astype(np.int64)
    fxr = px - x1.astype(np.float32)
    fyr = py - y1.astype(np.float32)
    inside = (x1 >= 0) & (y1 >= 0) & (x1 < w - 1) & (y1 < h - 1)
    xs, ys = np.where(inside, x1, 0), np.where(inside, y1, 0)
    one = E(np.float32(1.0))
    efx, efy = E(fxr), E(fyr)
    a00, a01, a10, a11 = (one - efx) * (one - efy), efx * (one - efy), (one - efx) * efy, efx * efy
    r0 = [E(R0[k]) for k in range(5)]
    s = []
    for k in range(5):
        P = np.asarray(R1[k], np.float32)
        s.append(a00 * E(P[ys, xs]) + a01 * E(P[ys, xs + 1]) + a10 * E(P[ys + 1, xs]) + a11 * E(P[ys + 1, xs + 1]))
    zero = E(np.zeros((h, w)))
    r2 = E.where(inside, s[0], zero)
    r3 = E.where(inside, s[1], zero)
    r4 = E.where(inside, (r0[2] + s[2]).scale2(0.5), r0[2])
    r5 = E.where(inside, (r0[3] + s[3]).scale2(0.5), r0[3])
    r6 = E.where(inside, (r0[4] + s[4]).scale2(0.25), r0[4].scale2(0.5))
    r2 = (r0[0] - r2).scale2(0.5)
    r3 = (r0[1] - r3).scale2(0.5)
    edx, edy = E(fx), E(fy)
    r2 = r2 + (r4 * edy + r6 * edx)
    r3 = r3 + (r6 * edy + r5 * edx)
    cb = lambda i: E(C_BORDER[np.minimum(i, 5)])  # noqa: E731
    scale = cb(xx) * cb(yy) * cb(w - xx - 1) * cb(h - yy - 1)
    r2, r3, r4, r5, r6 = (r * scale for r in (r2, r3, r4, r5, r6))
    return [r4 * r4 + r6 * r6, (r4 + r5) * r6, r5 * r5 + r6 * r6, r4 * r2 + r6 * r3, r6 * r2 + r5 * r3]


def update_matrices(fx, fy, R0, R1):
    """B.4: M0 .. M4 from the flow and the expansions R0 (frame a), R1 (frame b), each a sequence of five planes"""
    return [m.out() for m in _update_matrices_e(fx, fy, R0, R1)]


def box_mean(M, ksize=13):
    """B.5 box mean of each plane, index-clamped, vertical sums first, then x (1 / ksize^2) in fp32"""
    half = ksize // 2
    area_inv = E(np.float32(1.0) / np.float32(ksize * ksize))
    out = []
    for P in M:
        P = np.asarray(P, np.float32)
        h, w = P.shape
        yi, xi = np.arange(h), np.arange(w)
        acc = E(P)
        for j in range(1, half + 1):
            acc = acc + (E(P[np.maximum(yi - j, 0)]) + E(P[np.minimum(yi + j, h - 1)]))
        v = acc
        acc = v
        for j in range(1, half + 1):
            acc = acc + (v[:, np.maximum(xi - j, 0)] + v[:, np.minimum(xi + j, w - 1)])
        out.append(acc * area_inv)
    return out


RCP_REL = 4 * U  # rcp.approx.f32 (default build): 2 ulp; the strict build divides correctly rounded


def solve(b):
    """B.5 2x2 solve from five E planes (g11, g12, g22, h1, h2): (flow x, flow y) as (value, bound)"""
    g11, g12, g22, h1, h2 = b
    D = g11 * g22 - g12 * g12 + E(np.float32(1e-3))
    eD = D.bound()
    out = []
    for N in (g11 * h2 - g12 * h1, g22 * h1 - g12 * h2):
        eN = N.bound()
        den = np.abs(D.v) - eD
        q = np.abs(N.v) + eN
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(den > 0, (eN + np.abs(N.v) * eD / np.abs(D.v)) / den + q / den * ((1 + RCP_REL) * (1 + U) - 1), np.inf)
        out.append((N.v / D.v, e + 2 * TINY))
    return out


def update_flow(M):
    """orc_farn_update_flow alone: the 2x2 solve on fp32 box means"""
    return solve([E(np.asarray(p, np.float32)) for p in M])


def iteration(M, R0, R1, fx_at=None, fy_at=None, ksize=13):
    """one iteration: box mean -> solve (fx, fy), and M' = update_matrices evaluated at the flow (fx_at, fy_at) — the flow the
    device returned, so that a last-bit difference in the flow cannot move a gather into the next cell"""
    fx, fy = solve(box_mean(M, ksize))
    Mp = update_matrices(fx_at, fy_at, R0, R1) if fx_at is not None else None
    return fx, fy, Mp


def flow_init(pfx, pfy, lw, lh, pyr_scale=0.5):
    """level start: bilinear resize (CUDA convention) of the coarser flow to lw x lh, times (float)(1 / pyr_scale)"""
    out = []
    for P in (pfx, pfy):
        P = np.asarray(P, np.float32)
        ph, pw = P.shape
        sx, x1, xa, xb = _resize_coords(lw, pw, np.float32(1.0 / (lw / pw)))
        sy, y1, ya, yb = _resize_coords(lh, ph, np.float32(1.0 / (lh / ph)))
        b = [[E(P[np.ix_(r, c)]) for c in (xa, xb)] for r in (ya, yb)]
        out.append(_bilinear4(b, sx[None, :], x1[None, :], sy[:, None], y1[:, None]).scale2(1.0 / pyr_scale).out())
    return out
