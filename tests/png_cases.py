"""Images for the PNG encoder tests: probe sizes and contents, streams with runs of chosen lengths, and noise whose stream
has an exact number of literals."""
import numpy as np

# (h, w)
PROBE_SIZES = [(h, w) for h in range(1, 10) for w in range(1, 10)] + [
    (16, 16), (32, 32), (45, 80), (64, 64), (73, 74), (90, 91), (128, 128), (256, 340), (720, 1280), (1080, 1920), (1, 1920),
    (1920, 1), (1080, 7)]
CONTENTS = ("noise", "constant", "smooth", "mixed")
# h x (1 + 3 w) = 16383 k: the stream fills k deflate blocks exactly (129 x 127 = 16383)
BLOCK_EDGE_SIZES = [(129, 42), (258, 42), (387, 42)]


def image(kind, h, w, seed=0):
    rng = np.random.default_rng(seed + 7919 * h + w)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), np.uint8)
    if kind == "constant":
        return np.full((h, w, 3), 77, np.uint8)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    smooth = np.stack([128 + 40 * np.sin(xx / 37 + yy / 53), 128 + 30 * np.cos(yy / 29), np.where(yy <= h // 2, 5, 9)], -1)
    smooth = np.round(smooth).astype(np.uint8)
    if kind == "smooth":
        return smooth
    if kind == "mixed":  # half constant, half noise
        m = rng.integers(0, 256, (h, w, 3), np.uint8)
        m[: h // 2] = 9
        return m
    raise ValueError(kind)


def image_from_stream(sub, h, w):
    """The BGR image whose SUB-filtered scanlines (filter bytes excluded) are `sub` (uint8 [h, 3 w])."""
    rgb = np.cumsum(sub.reshape(h, w, 3).astype(np.int64), axis=1) % 256
    return np.ascontiguousarray(rgb[:, :, ::-1].astype(np.uint8))


def literal_noise(h, w, seed=0):
    """Noise whose scanline stream (filter bytes included) never has four equal bytes in a row: every symbol is a literal."""
    rng = np.random.default_rng(seed)
    while True:
        sub = rng.integers(0, 256, (h, 3 * w), np.uint8)
        raw = np.concatenate([np.ones((h, 1), np.uint8), sub], 1).ravel()
        same = raw[1:] == raw[:-1]
        if not (same[:-2] & same[1:-1] & same[2:]).any():
            return image_from_stream(sub, h, w)


def run_image(n):
    """One row whose stream holds a run of exactly n zero bytes after the first pixel: SUB of a constant row is zero past the
    first pixel, and a zero B (G) of the first pixel lengthens the run by one (two)."""
    extra = n % 3
    w = (n - extra) // 3 + 1
    first = [(50, 60, 70), (50, 60, 0), (50, 0, 0)][extra]  # R, G, B
    return np.tile(np.array(first[::-1], np.uint8), (1, w, 1))


def ramp(h, w):
    """Every SUB byte and every filter byte is 1: one run across all scanlines."""
    return image_from_stream(np.ones((h, 3 * w), np.uint8), h, w)


def rle_parse(raw):
    """deflate_rle's greedy parse: literal, or a match at distance 1 of min(run left, 258) when the next three bytes equal the
    previous one."""
    out, p, n = [], 0, len(raw)
    while p < n:
        if p > 0 and n - p >= 3 and raw[p] == raw[p + 1] == raw[p + 2] == raw[p - 1]:
            q = p
            while q < n and q - p < 258 and raw[q] == raw[p - 1]:
                q += 1
            out.append((q - p, 1))
            p = q
        else:
            out.append(raw[p])
            p += 1
    return out
