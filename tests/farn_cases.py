"""Inputs of the Farneback stage tests, the oracle's building blocks chained as the engine chains its kernels, and the
checks every stage test makes.

Shared by tests/test_farneback_reference_cpu.py (oracle vs the float64 bounds of tests/farn_ref64.py),
tests/test_farneback_kernels_gpu.py (kernels vs the oracle and vs the float64 bounds) and tests/test_farn_window_gpu.py
(the B.7 kernels vs tests/farn_restate.py and vs the float64 bounds)."""
import numpy as np

from denseflow_b200 import synth

# frames whose every pyramid level is checked (1080p has six levels, smoothing kernels up to 79 taps; 340x256 ends at 42x32;
# 131x97 rounds half to even to 66x48)
FRAME_SHAPES = [(1920, 1080), (1280, 720), (340, 256), (131, 97)]
# iteration / update_matrices planes (w, h): no interior tile at all and interior tiles of the 32 x 16 iteration tiling, last
# tiles one column or row wide, odd widths (the 2-pixel path clamps both pixels onto w - 1)
ITER_W = [32, 33, 40, 47, 64, 65, 72, 97]
ITER_H = [32, 33, 37, 38, 48, 49]
ITER_SHAPES = [(w, h) for w in ITER_W for h in ITER_H]
# frames and planes below the 32-px level cut (tests/geometry_cases.py): the 13-tap box and the 11-tap polynomial window
# wider than the image below 13, one 32 x 16 tile, a TMA window of 48 floats from x0 - 8 holding both border patches at w <= 8
SMALL_FRAMES = [(1, 1), (2, 1), (1, 3), (3, 2), (4, 4), (5, 7), (8, 8), (8, 1), (1, 8), (12, 5), (13, 13), (16, 9), (17, 31),
                (31, 31), (33, 31), (31, 63), (1, 200), (200, 2)]
SMALL_W = [1, 2, 3, 4, 5, 7, 8, 9, 12, 13, 16, 17, 31]
SMALL_H = [1, 2, 3, 5, 8, 13, 16, 17, 31]
ITER_SMALL = sorted({(w, SMALL_H[(3 * i + j) % len(SMALL_H)]) for i, w in enumerate(SMALL_W) for j in range(3)} |
                    {(1, 1), (8, 8), (13, 13), (31, 31)})
FLOW_KINDS = ["smooth", "iid", "edges", "far"]


def frame_f32(w, h, seed=0):
    return synth.pair(h, w, seed)[0].astype(np.float32)


def flow(kind, w, h, seed):
    """flow fields that drive update_matrices into each of its branches"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    if kind == "smooth":  # neighbours' tap cells are adjacent: the shared-gather branch of the 2-pixel path
        fx = 1.7 * np.sin(yy / 9.0 + seed) + 0.6 * np.cos(xx / 23.0) + 0.3
        fy = -1.2 * np.cos(xx / 11.0 + seed) + 0.4 * np.sin(yy / 17.0)
    elif kind == "iid":  # independent per pixel: the fallback branch
        fx = rng.normal(0.0, 2.5, (h, w))
        fy = rng.normal(0.0, 2.5, (h, w))
    elif kind == "edges":  # x1 = x + dx and y1 = y + dy exactly at -1, 0, n-2, n-1, fractional parts exactly 0
        tx = np.array([-1, 0, w - 2, w - 1])[rng.integers(0, 4, (h, w))]
        ty = np.array([-1, 0, h - 2, h - 1])[rng.integers(0, 4, (h, w))]
        fx = tx - xx
        fy = ty - yy
        keep = rng.random((h, w)) < 0.25  # some pixels keep a sub-pixel flow between the edge taps
        fx = np.where(keep, rng.uniform(-0.9, 0.9, (h, w)), fx)
        fy = np.where(keep, rng.uniform(-0.9, 0.9, (h, w)), fy)
    elif kind == "far":  # far outside the image, some of it
        fx = rng.uniform(-900.0, 900.0, (h, w)) * (rng.random((h, w)) < 0.5) + rng.normal(0, 1, (h, w))
        fy = rng.uniform(-900.0, 900.0, (h, w)) * (rng.random((h, w)) < 0.5) + rng.normal(0, 1, (h, w))
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(fx, np.float32), np.ascontiguousarray(fy, np.float32)


def stack(planes):
    """the planes of several pairs as one launch's input plane, pair after pair down the rows"""
    return np.ascontiguousarray(np.concatenate(planes, axis=0))


def split(a, n):
    """one launch's output plane back into its n pairs' planes"""
    return np.split(a, n, axis=0)


def within(name, got, ref):
    """every element of `got` within the float64 bound: ref = (float64 value, bound)"""
    v, b = ref
    bad = ~(np.abs(got.astype(np.float64) - v) <= b)
    assert not bad.any(), "%s: %d elements outside the float64 bound, first at %s: got %r, float64 %r, bound %r" % (
        name, bad.sum(), tuple(np.argwhere(bad)[0]), got[bad][0], v[bad][0], b[bad][0])


def check(variant, name, got, exact, ref64):
    """strict build: `got` equals `exact` by value; default build: `got` within the float64 bound `ref64`"""
    if variant == "strict":
        diff = got != exact
        assert not diff.any(), "%s: %d elements differ, first at %s: got %r, want %r" % (
            name, diff.sum(), tuple(np.argwhere(diff)[0]), got[diff][0], exact[diff][0])
    else:
        within(name, got, ref64)


class Oracle:
    """the oracle's Farneback building blocks on numpy planes (R / M: float32 [5, h, w])"""

    def __init__(self, pyoracle):
        self.po = pyoracle
        self.L = pyoracle.lib()

    def levels(self, w, h, **kw):
        return self.po.farn_levels(w, h, self.po.farn_params(**kw) if kw else None)

    def level_image(self, frame, k, **kw):
        """orc_farn_gaussian_blur(smooth_k, sigma_k) then orc_resize_linear(CUDA) with the engine's rfx / rfy"""
        h, w = frame.shape
        lv = self.levels(w, h, **kw)
        lw, lh, smooth, sigma = lv[len(lv) - 1 - k]
        blurred = np.empty((h, w), np.float32)
        self.L.orc_farn_gaussian_blur(np.ascontiguousarray(frame, np.float32), w, h, smooth, sigma, blurred)
        img = np.empty((lh, lw), np.float32)
        rfx, rfy = np.float32(1.0 / (lw / w)), np.float32(1.0 / (lh / h))
        self.L.orc_resize_linear(blurred, w, h, img, lw, lh, rfx, rfy, self.po.RESIZE_CUDA)
        return img, (lw, lh, smooth, sigma)

    def poly_exp(self, img, sigma=1.1):
        h, w = img.shape
        R = np.empty((5, h, w), np.float32)
        self.L.orc_farn_poly_exp(np.ascontiguousarray(img, np.float32), w, h, 5, sigma, R)
        return R

    def update_matrices(self, fx, fy, R0, R1):
        h, w = fx.shape
        M = np.empty((5, h, w), np.float32)
        self.L.orc_farn_update_matrices(np.ascontiguousarray(fx), np.ascontiguousarray(fy), np.ascontiguousarray(R0),
                                        np.ascontiguousarray(R1), w, h, M)
        return M

    def box_filter5(self, M):
        h, w = M.shape[1:]
        B = np.empty_like(M)
        self.L.orc_farn_box_filter5(np.ascontiguousarray(M), w, h, 13, B)
        return B

    def update_flow(self, B):
        h, w = B.shape[1:]
        fx = np.empty((h, w), np.float32)
        fy = np.empty((h, w), np.float32)
        self.L.orc_farn_update_flow(np.ascontiguousarray(B), w, h, fx, fy)
        return fx, fy

    def iteration(self, M, R0, R1, rebuild):
        """box mean -> solve -> (if rebuild) update_matrices: fx, fy, M' (None without rebuild)"""
        fx, fy = self.update_flow(self.box_filter5(M))
        return fx, fy, (self.update_matrices(fx, fy, R0, R1) if rebuild else None)

    def flow_init(self, pfx, pfy, lw, lh):
        ph, pw = pfx.shape
        rfx, rfy = np.float32(1.0 / (lw / pw)), np.float32(1.0 / (lh / ph))
        out = []
        for p in (pfx, pfy):
            o = np.empty((lh, lw), np.float32)
            self.L.orc_resize_linear(np.ascontiguousarray(p, np.float32), pw, ph, o, lw, lh, rfx, rfy, self.po.RESIZE_CUDA)
            out.append(o * np.float32(1.0 / 0.5))
        return out

    def expansions(self, w, h, seed):
        """R of two real frames (full-resolution level image -> polynomial expansion)"""
        a, b, _ = synth.pair(h, w, seed)
        return [self.poly_exp(self.level_image(f.astype(np.float32), 0)[0]) for f in (a, b)]

    def pair_case(self, w, h, seed, kind):
        """one pair of the iteration tests: R0, R1 of real frames, M = update_matrices at a flow of `kind` (PSD, like the
        engine's)"""
        R0, R1 = self.expansions(w, h, seed)
        fx, fy = flow(kind, w, h, seed)
        return R0, R1, self.update_matrices(fx, fy, R0, R1)
