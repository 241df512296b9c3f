"""Frame geometries at the thresholds where the engines change behaviour, shared by the stage tests, the CPU tests of the
oracle's building blocks and the end-to-end sweep of tests/test_geometry_gpu.py.  All shapes are (w, h).

Where the constants come from:
* TV-L1 pyramid: level s is round-half-even(0.8 * level s - 1) and a level narrower or shorter than 16 px is dropped
  (Tvl1::level_geometry), so below 20 x 20 the pyramid is one level;
* Farneback pyramid: levels stop once w * 0.5^k or h * 0.5^k drops under 32 (Farneback::levels_for), depth 5;
* fused TV-L1 tile 128 x 64, 4 rows per warp band, halo kk <= 8 rows and (kk + 3) & ~3 columns: with h < 4 one warp band
  covers the whole image and with h <= 2 * kk the halo is taller than the image;
* four-pixel groups of the u8 -> f32 conversion and of the TV-L1 primal row: with w < 4 one group holds both column 0 and
  column w - 1;
* Farneback iteration tile 32 x 16 and its TMA window of 48 floats from x0 - 8: with w <= 8 both border patches fall in
  one window;
* Farneback box window 13 (half-width 6) and the polynomial window of poly_n 5 (11 taps): below 13 px both are wider than
  the image.
"""

TV_SCALE, TV_MIN, TV_SCALES = 0.8, 16, 5
FARN_SCALE, FARN_MIN, FARN_DEPTH = 0.5, 32, 5


def tvl1_levels(w, h):
    """number of TV-L1 pyramid levels at the default parameters (Python's round() is half-to-even like std::nearbyint)"""
    n, cw, ch = 1, w, h
    for _ in range(1, TV_SCALES):
        cw, ch = round(cw * TV_SCALE), round(ch * TV_SCALE)
        if cw < TV_MIN or ch < TV_MIN:
            break
        n += 1
    return n


def farn_levels(w, h):
    """number of Farneback pyramid levels at the default parameters"""
    k, scale = 0, 1.0
    while k < FARN_DEPTH:
        scale *= FARN_SCALE
        if w * scale < FARN_MIN or h * scale < FARN_MIN:
            break
        k += 1
    return k + 1


def level_cuts(levels, limit=2200):
    """square sizes n at which levels(n, n) != levels(n - 1, n - 1)"""
    return [n for n in range(2, limit) if levels(n, n) != levels(n - 1, n - 1)]


TINY = [(w, h) for h in range(1, 9) for w in range(1, 9)]                       # every w and h in 1..8
AROUND = [12, 13, 15, 16, 17, 31, 32, 33]                                        # box 13, TV-L1 cut 16, Farneback cut 32
SQUARES = [(n, n) for n in AROUND]
STRIPS = [(1, 1920), (1920, 1), (7, 1080), (1080, 7)]
LARGE = [(3840, 2160), (2047, 1151)]
# below each level cut and at it: the level count changes between the two
TVL1_CUTS = [s for n in level_cuts(tvl1_levels) for s in ((n - 1, n), (n, n))]
FARN_CUTS = [s for n in level_cuts(farn_levels) for s in ((n - 1, n), (n, n))]

# the stage tests (cheap): every small plane, thin strips
STAGE_SMALL = TINY + [(w, h) for w in (12, 13, 15) for h in (1, 2, 3, 5, 12, 13, 15)] + [(15, 9), (9, 15), (11, 4), (4, 11)]
STAGE_STRIPS = [(1, 400), (400, 1), (2, 257), (257, 3), (7, 300), (300, 7)]


def e2e(algorithm):
    """the end-to-end sweep, largest first (one handle created at 3840 x 2160 serves it in this order): the level cuts of
    the algorithm (the Farneback ones up to 512, above that the cost is the oracle's), the squares around the tile and
    window sizes, a selection of the tiny frames and the thin strips"""
    cuts = TVL1_CUTS if algorithm == "tvl1" else [s for s in FARN_CUTS if s[1] <= 512]
    tiny = [(8, 8), (7, 5), (5, 7), (4, 4), (8, 1), (1, 8), (3, 2), (2, 3), (4, 1), (1, 4), (2, 2), (2, 1), (1, 2), (1, 1)]
    shapes = LARGE + STRIPS + cuts + SQUARES + tiny
    return sorted(dict.fromkeys(shapes), key=lambda s: -s[0] * s[1])


# uint8 INTER_LINEAR resize, (source (w, h), destination (w, h)): one-pixel sources and destinations, single rows and columns,
# upscales from one pixel, long thin strips, and the decode stage's 1920 x 1080 -> 455 x 256
RESIZE_CASES = [((1, 1), (1, 7)), ((1, 1), (7, 1)), ((1, 1), (5, 3)), ((7, 1), (1, 1)), ((1, 7), (1, 1)), ((1, 7), (3, 7)),
                ((7, 1), (7, 4)), ((2, 2), (1, 1)), ((2, 2), (3, 3)), ((3, 2), (8, 5)), ((13, 2000), (7, 300)), ((2000, 13), (300, 7)),
                ((13, 2000), (1, 1)), ((2000, 13), (2001, 1)), ((1, 2000), (1, 13)), ((1920, 1080), (455, 256)), ((33, 17), (1, 17)),
                ((17, 33), (17, 1)), ((5, 5), (160, 120))]
