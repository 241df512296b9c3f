"""Images whose zlib streams reach the edges of zlib's deflate that the GPU PNG encoder (denseflow_b200/csrc/png_deflate.cuh,
png_encode.cu) restates: Huffman trees deeper than their length limit, fake tree nodes, exact ties in the stored / fixed /
dynamic choice, a block flush inside a run, the window size declared in the zlib header and the 8 KB IDAT chunk edges.
Every case names the edge it is built to reach; tests/test_png_deflate_cpu.py asserts, through zlib's own stream
(tests/inflate_trace.py) and the size model (tests/zlib_sizes.py), that it does reach it, and tests/test_png_deflate_gpu.py
encodes it.  Parameters found by search are committed here, so every case is deterministic."""
import numpy as np

import png_cases as PC
import png_restate as P

FIB = [1, 1]
while len(FIB) < 30:
    FIB.append(FIB[-1] + FIB[-2])


def image_from_raw(raw, h, w):
    """The BGR image whose filtered scanline stream (filter bytes included) is raw."""
    rows = np.frombuffer(bytes(raw), np.uint8).reshape(h, 1 + 3 * w)
    assert (rows[:, 0] == (0 if w == 1 else 1)).all(), "filter bytes"
    if w == 1:  # filter NONE: the bytes are R, G, B
        return np.ascontiguousarray(rows[:, 1:][:, ::-1].reshape(h, 1, 3))
    return PC.image_from_stream(rows[:, 1:], h, w)


def no_matches(raw):
    """True when no byte equals the three before it: Z_RLE then emits every byte as a literal."""
    a = np.frombuffer(bytes(raw), np.uint8)
    same = a[1:] == a[:-1]
    return not (same[:-2] & same[1:-1] & same[2:]).any()


def spread(counts):
    """counts[v] bytes of each value v, every value's occurrences evenly spaced over the result"""
    keys = np.concatenate([(np.arange(c) + 0.5) / c for c in counts.values()])
    vals = np.concatenate([np.full(c, v, np.uint8) for v, c in counts.items()])
    return vals[np.argsort(keys, kind="stable")].tobytes()


def literal_histogram(counts, h, w):
    """The image whose scanline stream holds exactly counts[v] bytes of each value v (the h filter bytes included), with no
    run of four equal bytes: every symbol is a literal, so the histogram of the stream's single (or first) block is counts
    plus END_BLOCK's 1."""
    f = 0 if w == 1 else 1
    assert sum(counts.values()) == h * (1 + 3 * w) and counts.get(f, 0) >= h
    rest = dict(counts)
    rest[f] -= h
    body = np.frombuffer(spread({v: c for v, c in rest.items() if c}), np.uint8).reshape(h, 3 * w)
    raw = np.concatenate([np.full((h, 1), f, np.uint8), body], 1).tobytes()
    assert no_matches(raw)
    return image_from_raw(raw, h, w)


def _fit_top(counts, top, extra=0):
    """raise counts[top] by 0..2 so the stream (extra bytes besides the counts) fills one scanline: 1 + 3 w bytes"""
    counts[top] += (1 - sum(counts.values()) - extra) % 3
    return (sum(counts.values()) + extra - 1) // 3


def chain_values(k, avoid=(1,)):
    """k distinct byte values scattered over 0..255, none of them in avoid"""
    out = [v for v in (np.arange(256) * 97 + 5) % 256 if v not in avoid]
    return [int(v) for v in out[:k]]


def fibonacci(depth):
    """A one-row image whose single block's literal tree is a chain depth deep before zlib limits it to 15 bits: the filter
    byte (value 1) and END_BLOCK are the chain's two 1s, then depth - 1 values with counts 2, 3, 5, 8, ..."""
    counts = {1: 1}
    vals = chain_values(depth - 1)
    for v, c in zip(vals, FIB[2:depth + 1]):
        counts[v] = c
    w = _fit_top(counts, vals[-1])
    return literal_histogram(counts, 1, w)


LUCAS = [2, 1]
while len(LUCAS) < 30:
    LUCAS.append(LUCAS[-1] + LUCAS[-2])


def lucas(depth):
    """The cheapest chain under zlib's depth tie-break: three 1s (the filter byte, END_BLOCK and one value), then depth - 2
    values with the Lucas counts 3, 4, 7, 11, 18, ...  The two 1s merge first, the third 1 joins that node, and from there
    each equal-count tie between a leaf and the chain's node goes to the shallower leaf, so the tree stays a chain.  Depth
    19 costs 15 126 symbols (Fibonacci counts need 17 710), so it fits one block of 16 383."""
    counts = {1: 1}
    vals = chain_values(depth - 1)
    for v, c in zip(vals, [1] + LUCAS[2:depth]):
        counts[v] = c
    w = _fit_top(counts, vals[-1])
    return literal_histogram(counts, 1, w)


def _noise_bytes(n, seed, first=None):
    """n random bytes with no run of four equal bytes (first: the stream's first byte, which they must continue)"""
    rng = np.random.default_rng(seed)
    while True:
        b = rng.integers(0, 256, n, np.uint8).tobytes()
        if no_matches((first or b"") + b):
            return b


def deep_middle_block(depth=17):
    """Three literal blocks: noise, a Fibonacci chain depth deep (END_BLOCK and one value are its 1s) and noise; the deep
    block is neither the first nor the last one.  The chain's two largest counts share what fills the block to 16 383
    symbols, which keeps it a chain and keeps any value under half of the block."""
    vals = chain_values(depth, avoid=())
    counts = dict(zip(vals, FIB[1:depth + 1]))
    fill = 16383 - sum(counts.values())
    counts[vals[-2]] += fill // 2
    counts[vals[-1]] += fill - fill // 2
    mid = spread(counts)
    for seed in range(100):  # a partial last block of 8002 bytes: 2 x 16383 + 8002 = 1 + 3 w
        raw = b"\x01" + _noise_bytes(16382, seed, b"\x01") + mid + _noise_bytes(8002, seed + 1)
        if no_matches(raw):
            return image_from_raw(raw, 1, (len(raw) - 1) // 3)
    raise AssertionError("no seed found")


# match lengths of the runs deep_with_lengths places: two of length code 265 (one extra bit), three of code 279 (four)
CHAIN_MATCHES = {265: (11, 12), 279: (99, 106, 114)}


def deep_with_lengths(depth=17):
    """A Fibonacci literal / length chain depth deep whose deepest symbols after END_BLOCK and the filter byte are two length
    codes with extra bits: length code 265 (count 2), 279 (count 3), then the byte the five runs repeat (count 5, every run's
    first byte is a literal), then literals."""
    run_byte = 200
    vals = chain_values(depth - 4, avoid=(1, run_byte))
    counts = {1: 1}
    for v, c in zip(vals, FIB[5:depth + 1]):
        counts[v] = c
    runs = [n + 1 for lens in CHAIN_MATCHES.values() for n in lens]
    w = _fit_top(counts, vals[-1], extra=sum(runs))
    body = bytearray(spread({v: c for v, c in counts.items() if v != 1}))
    step = len(body) // (len(runs) + 1)
    for i, n in reversed(list(enumerate(runs))):  # runs at evenly spaced positions; their neighbours are other bytes
        p = step * (i + 1)
        body[p:p] = bytes([run_byte]) * n
    raw = b"\x01" + bytes(body)
    assert len(raw) == 1 + 3 * w
    return image_from_raw(raw, 1, w)


# (values, ratio, top count, seed) of geometric literal histograms whose code-length tree is 8 deep before zlib limits it
# to 7 (found by searching seeds with tests/zlib_sizes.py)
GEOMETRIC = [(114, 0.805, 2703, 88), (190, 0.826, 2315, 109), (150, 0.879, 1464, 188)]


def geometric(nvals, ratio, top, seed):
    """literal_histogram of nvals byte values at random positions of 0..255, counts max(1, round(top * ratio^i))"""
    rng = np.random.default_rng(seed)
    vals = rng.permutation(256)[:nvals]
    counts = {int(v): max(1, int(round(top * ratio ** i))) for i, v in enumerate(vals)}
    counts[1] = counts.get(1, 0) + 1  # the filter byte
    w = _fit_top(counts, int(vals[0]))
    return literal_histogram(counts, 1, w)


def only_literal(v, h=40, w=30):
    """A stream whose only literal byte value is v, for v = 0 (width 1 and black: filter NONE) or v = 1 (every SUB byte and
    filter byte 1): the literal tree holds v, END_BLOCK and lengths, the distance tree distance 1 alone, which takes the
    `max_code < 2` fake-node branch.  No image has a stream whose only literal is 2 or more: every scanline starts with
    filter byte 0 or 1, and a later block that avoids it would need a run of over 4 MB within one row.  The `: 0` branch
    that such a stream would reach is taken by the empty final block instead (END_BLOCK alone, max_code 256)."""
    if v == 0:
        return np.zeros((h, 1, 3), np.uint8)
    assert v == 1
    return PC.ramp(h, w)


def no_match_block():
    """a small dynamic block without matches: the distance tree is empty, so build_tree adds two fake nodes"""
    counts = {1: 1, 2: 40, 3: 40, 4: 40, 5: 3, 6: 3}
    w = _fit_top(counts, 2)
    return literal_histogram(counts, 1, w)


def run_across_flush(where):
    """A long run whose symbols straddle the first block flush: the 16 383rd symbol is the run's first byte ("head"), its
    second 258-byte match ("match") or its first trailing literal ("tail").  The run is 777 bytes: a literal, three
    matches of 258 and two literals."""
    pre = {"head": 16382, "match": 16382 - 2, "tail": 16382 - 4}[where]
    run = b"\x07" * 777
    for seed in range(100):
        head = b"\x01" + _noise_bytes(pre - 1, seed, b"\x01")
        n_after = 3000 + (1 - (pre + 777 + 3000)) % 3
        raw = head + run + _noise_bytes(n_after, seed + 1)
        if head[-1] != 7 and raw[pre + 777] != 7 and no_matches(head) and no_matches(raw[pre + 777:]):
            return image_from_raw(raw, 1, (len(raw) - 1) // 3)
    raise AssertionError("no seed found")


def run_noise(w, alphabet, mean_run, seed):
    """One row of runs of random bytes below `alphabet`, of geometric lengths with mean mean_run: near-incompressible to
    highly compressible streams, whose stored, fixed and dynamic sizes cross"""
    rng = np.random.default_rng(seed)
    out, prev = bytearray(b"\x01"), 1
    while len(out) < 1 + 3 * w:
        v = int(rng.integers(0, alphabet))
        if v != prev:
            out += bytes([v]) * int(rng.geometric(1 / mean_run))
            prev = v
    return image_from_raw(bytes(out[:1 + 3 * w]), 1, w)


def stretched_run_noise(w, alphabet, mean_run, seed, stretch=0):
    """run_noise (alphabet <= 255) with a run of 36 + stretch bytes of 255 in its middle: one match of 35 + stretch, length
    code 273 (35..42, three extra bits) for stretch 0..7.  Stretching the run adds bytes to the block but changes no symbol
    code, so the block's dynamic and fixed sizes stay the same while its stored size grows; stretch is 0, 3 or 6 so the
    stream still fills one scanline."""
    assert alphabet <= 255 and stretch in (0, 3, 6)
    raw = P.scanlines(run_noise(w, alphabet, mean_run, seed))
    mid = len(raw) // 2
    raw = raw[:mid] + b"\xff" * (36 + stretch) + raw[mid:]
    return image_from_raw(raw, 1, (len(raw) - 1) // 3)


# (edge, parameters) of images whose single block sits on a block-choice tie or next to it (found by searching seeds with
# tests/zlib_sizes.py).  stored+k: stored_len + k == min(dynamic, fixed) size in bytes, stretched_run_noise parameters;
# fixed=dynamic+k: the fixed size is the dynamic size + k bytes, run_noise parameters.
STORED_TIES = [
    ("stored+3", (544, 248, 1.17, 348)),
    ("stored+4", (452, 240, 1.04, 625)),  # the tie: stored
    ("stored+5", (1858, 254, 1.04, 160)),
]
FIXED_TIES = [
    ("fixed=dynamic-1", (62, 99, 5.12, 149)),
    ("fixed=dynamic+0", (89, 107, 5.26, 135)),  # the tie: fixed
    ("fixed=dynamic+1", (76, 128, 5.11, 49)),
]


def tie_cases():
    return [(name, stretched_run_noise(*p)) for name, p in STORED_TIES] + [(name, run_noise(*p)) for name, p in FIXED_TIES]


def shapes_of_length(n,max_w=3840, max_h=2160):
    """(h, w) with h (1 + 3 w) = n, w >= 2"""
    return [(h, (n // h - 1) // 3) for h in range(1, max_h + 1) if n % h == 0 and (n // h - 1) % 3 == 0 and 2 <= (n // h - 1) // 3 <= max_w]


def window_cases():
    """(name, h, w): raw stream lengths of exactly 2^k for k = 8..14 (width 85: 256 bytes a row), the nearest reachable lengths
    on either side of each, and width 1 (filter NONE, 4 bytes a row) at 2^k for k = 8..13"""
    out = []
    for k in range(8, 15):
        out.append(("2^%d" % k, 1 << (k - 8), 85))
        for sign in (-1, 1):
            d = 1
            while not shapes_of_length((1 << k) + sign * d):
                d += 1
            h, w = shapes_of_length((1 << k) + sign * d)[0]
            out.append(("2^%d%+d" % (k, sign * d), h, w))
    for k in range(8, 14):
        out.append(("2^%d w1" % k, 1 << (k - 2), 1))
    return out


def window_image(h, w):
    return PC.image("smooth" if h * w > 64 else "noise", h, w, seed=h + w)


def zero_prefix(h, w, z, seed=0):
    """noise whose first z SUB bytes (filter bytes excluded) are zero"""
    sub = np.random.default_rng(seed).integers(0, 256, (h, 3 * w), np.uint8).ravel()
    sub[:z] = 0
    return PC.image_from_stream(sub.reshape(h, 3 * w), h, w)


# zlib stream length -> (h, w, z) of zero_prefix (found by searching z): 8192 k - 1, 8192 k, 8192 k + 1 for k = 1, 2.  At
# 8192 k + 1 the last IDAT chunk holds 1 byte.
IDAT_CASES = {8191: (48, 60, 551), 8192: (48, 60, 550), 8193: (48, 60, 549),
              16383: (92, 60, 311), 16384: (92, 60, 310), 16385: (92, 60, 309)}


def idat_image(target):
    h, w, z = IDAT_CASES[target]
    return zero_prefix(h, w, z)


def zlib_len(img):
    return len(P.zlib_stream(P.scanlines(img)))


def synthetic_flow(h=1080, w=1920, seed=2, amp=4.0):
    """A smooth flow field plus 0.05 px noise.  At 1920 x 1080 with the defaults, two of the 312 blocks of its packed image
    (-st=png) need the literal-tree repair (1.0 and seed 0 give one of 371, other seeds none)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    fx = amp * (np.sin(xx / 150 + 0.3) + np.cos(yy / 90)) + rng.normal(0, 0.05, (h, w))
    fy = amp * (np.cos(xx / 110) - np.sin(yy / 70 + 1)) + rng.normal(0, 0.05, (h, w))
    return np.stack([fx, fy], -1).astype(np.float32)


def cases():
    """(name, image, edge) of every single-image case; edge names what tests/test_png_deflate_cpu.py asserts it reaches"""
    out = [("fibonacci%d" % d, fibonacci(d), "lit_depth=%d" % d) for d in (16, 17, 18)]
    out.append(("lucas19", lucas(19), "lit_depth=19"))
    out.append(("deep_middle_block", deep_middle_block(), "lit_depth=17@1/3"))
    out.append(("deep_with_lengths", deep_with_lengths(), "lit_depth=17+lengths"))
    out += [("geometric%d" % i, geometric(*p), "bl_depth>=8") for i, p in enumerate(GEOMETRIC)]
    out.append(("only_literal0", only_literal(0), "dist_fake=[1],lits=[0]"))
    out.append(("only_literal1", only_literal(1), "dist_fake=[1],lits=[1]"))
    out.append(("no_matches", no_match_block(), "dist_fake=[0, 1]"))
    out.append(("empty_final_block", PC.literal_noise(129, 42), "lit_fake=[0]"))
    out += [(n, img, n) for n, img in tie_cases()]
    out += [("flush_at_run_" + wh, run_across_flush(wh), "flush@" + wh) for wh in ("head", "match", "tail")]
    out += [("window_" + n, window_image(h, w), "raw=%d" % (h * (1 + 3 * w))) for n, h, w in window_cases()]
    out += [("idat_%d" % t, idat_image(t), "zlen=%d" % t) for t in sorted(IDAT_CASES)]
    return out
