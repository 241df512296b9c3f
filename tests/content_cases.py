"""Gray frame pairs and one stream with the content of real videos, for the end-to-end tests of both engines.

synth.pair is a blurred-noise texture under a smooth motion of at most about 14 px: every pixel is textured and every
(scale, warp) of TV-L1 converges early.  Real inputs also have black bars, static shots, fades, cuts, fast pans, clipped
highlights, periodic patterns, occluding objects and flat sensor noise.  Each recipe below is deterministic (fixed seeds,
synth and cv2 only) and drives one of those regimes; tests/test_content_cpu.py asserts on the oracle that it still does.

Every recipe takes (w, h) and returns the pair (a, b) as uint8 [h, w] frames:
  synth            synth.pair: the content every other end-to-end test uses
  letterbox        synth.pair with rows [0, h/8) and [h - h/8, h) black in both frames (or bars of `bar` rows)
  pillarbox        synth.pair with columns [0, w/8) and [w - w/8, w) at 16 in both frames
  static           (a, a)
  fade_half        (a, a // 2)
  fade_black       (a, 0)
  fade_from_black  (0, a)
  cut              synth.noise_pair: b is an independent texture
  pan              two crops of one larger texture 40 px apart horizontally (the content moves 40 px to the right)
  pan_diagonal     the same 40 px right and 24 px down
  clipped          clip(3a - 255) of both frames of synth.pair: blown-out highlights and crushed shadows
  checkerboard     8 px squares of 0 and 255; b is cv2.warpAffine of a by (2.5, 1.25), cubic, reflect border (the cubic
                   overshoot saturates, so about 40 % of b is exactly flat)
  square           a textured square of a third of the frame moving 6 px right over a static textured background (the
                   class whose TV-L1 run has pixels with 0 < g <= FLT_EPSILON and |rho| <= l_t * g, where the reference's
                   primal step picks 0 and the default build sign(-rho) * l_t)
  noise            flat gray 128 with independent uniform integer noise in [-2, 2] per frame
"""
import numpy as np

from denseflow_b200 import synth

CLASSES = ["synth", "letterbox", "pillarbox", "static", "fade_half", "fade_black", "fade_from_black", "cut", "pan", "pan_diagonal",
           "clipped", "checkerboard", "square", "noise"]
SMALL_CLASSES = ["letterbox", "static", "fade_black", "fade_from_black", "cut", "pan", "checkerboard", "square"]
SIZE = (340, 256)    # the benchmark's clip
SMALL = (131, 97)    # odd sizes: partial tiles and odd level sizes
HD = (1920, 1080)
HD_LETTERBOX_BAR = 140  # 2.39:1 content in a 16:9 frame

# the oracle's regimes (tests/test_content_cpu.py): every (scale, warp) of TV-L1 at its minimum of 2 iterations, or at the
# cap of 300
AT_MINIMUM = ["static", "fade_black"]
AT_CAP = ["fade_half", "fade_from_black", "cut", "pan", "pan_diagonal"]


def _synth(w, h, seed=0):
    a, b, _ = synth.pair(h, w, seed)
    return a, b


def letterbox(w, h, bar=None):
    a, b = _synth(w, h, 1)
    bar = h // 8 if bar is None else bar
    for f in (a, b):
        f[:bar] = 0
        f[h - bar:] = 0
    return a, b


def pillarbox(w, h):
    a, b = _synth(w, h, 2)
    bar = w // 8
    for f in (a, b):
        f[:, :bar] = 16
        f[:, w - bar:] = 16
    return a, b


def pan(w, h, dx=40, dy=0, seed=3):
    """frame a shows the texture at (dx, dy), frame b at (0, 0): the flow of a -> b is (+dx, +dy) everywhere"""
    big = _synth(w + dx, h + dy, seed)[0]
    return np.ascontiguousarray(big[dy:dy + h, dx:dx + w]), np.ascontiguousarray(big[:h, :w])


def checkerboard(w, h):
    import cv2
    yy, xx = np.mgrid[0:h, 0:w]
    a = (((xx // 8) + (yy // 8)) % 2 * 255).astype(np.uint8)
    m = np.float32([[1, 0, 2.5], [0, 1, 1.25]])
    b = cv2.warpAffine(a, m, (w, h), flags=cv2.INTER_CUBIC, borderMode=cv2.BORDER_REFLECT)
    return a, b


def square(w, h, dx=6):
    bg = _synth(w, h, 5)[0]
    fg = _synth(w, h, 6)[0]
    s = max(min(w, h) // 3, 4)
    x0, y0 = (w - s) // 2 - dx // 2, (h - s) // 2
    a, b = bg.copy(), bg.copy()
    a[y0:y0 + s, x0:x0 + s] = fg[:s, :s]
    b[y0:y0 + s, x0 + dx:x0 + dx + s] = fg[:s, :s]
    return a, b


def noise(w, h):
    rng = np.random.default_rng(8)
    return tuple((128 + rng.integers(-2, 3, (h, w))).astype(np.uint8) for _ in range(2))


def pair(name, w, h):
    """(a, b) of class `name` at w x h"""
    if name == "synth":
        return _synth(w, h)
    if name == "letterbox":
        return letterbox(w, h)
    if name == "pillarbox":
        return pillarbox(w, h)
    if name == "pan":
        return pan(w, h)
    if name == "pan_diagonal":
        return pan(w, h, 40, 24)
    if name == "checkerboard":
        return checkerboard(w, h)
    if name == "square":
        return square(w, h)
    if name == "noise":
        return noise(w, h)
    if name == "cut":
        return synth.noise_pair(h, w, 4)
    a = _synth(w, h, 11)[0]  # a texture whose fades drive TV-L1's flow past the frame width at both test sizes
    if name == "static":
        return a, a.copy()
    if name == "fade_half":
        return a, a // 2
    if name == "fade_black":
        return a, np.zeros_like(a)
    if name == "fade_from_black":
        return np.zeros_like(a), a
    if name == "clipped":
        return tuple(np.clip(3 * f.astype(np.int32) - 255, 0, 255).astype(np.uint8) for f in _synth(w, h, 9))
    raise KeyError(name)


def cases():
    """(name, w, h) of every pair the GPU tests pin: every class at 340 x 256, a subset at 131 x 97, and at 1920 x 1080 the
    2.39:1 letterbox and the pan"""
    return ([(c,) + SIZE for c in CLASSES] + [(c,) + SMALL for c in SMALL_CLASSES] +
            [("letterbox_239",) + HD, ("pan",) + HD])


def case_pair(name, w, h):
    if name == "letterbox_239":
        return letterbox(w, h, HD_LETTERBOX_BAR)
    return pair(name, w, h)


# the stream: its pairs at step 1 take turns between the classes below and the transition from one class's second frame to
# the next class's first frame (a cut, a fade from black or a static pair)
STREAM_CLASSES = ["static", "cut", "synth", "fade_black", "pan", "letterbox", "checkerboard", "fade_half", "square"]


def stream(w=SIZE[0], h=SIZE[1]):
    """uint8 [2 * len(STREAM_CLASSES), h, w]: the frames a0, b0, a1, b1, ... of the classes' pairs"""
    return np.stack([f for c in STREAM_CLASSES for f in pair(c, w, h)])


def flat_fraction(oracle, frame):
    """share of the pixels whose TV-L1 "grad" g = I1x^2 + I1y^2 is <= FLT_EPSILON where the warp is the identity (the finest
    level at zero flow: the warp's taps collapse onto the centre pixel, so I1wx = I1x and I1wy = I1y of the second frame)"""
    f = np.ascontiguousarray(frame, np.float32)
    h, w = f.shape
    gx, gy = np.empty_like(f), np.empty_like(f)
    oracle.lib().orc_centered_gradient(f, w, h, gx, gy)
    g = gx * gx + gy * gy
    return float(np.mean(g <= np.finfo(np.float32).eps))
