"""A numpy / pure-Python restatement of `cv2.imdecode(buf, IMREAD_COLOR)` (libjpeg-turbo's default decompression: islow IDCT,
fancy upsampling, YCbCr -> BGR) for the subset of JPEG files the GPU decoder accepts, so its stages can be checked one at a
time: `parse` (markers, tables), `coefficients` (entropy decode: natural order, absolute DC), `idct_planes` and `to_bgr`.

The subset, and the two exceptions it raises:
* baseline / extended sequential Huffman (SOF0, SOF1), 8-bit samples, one scan holding every component;
* 1 component, or 3 that libjpeg treats as YCbCr (JFIF marker, Adobe transform 1, or component ids 1-2-3);
* chroma sampled 1 x 1, luma h, v in {1, 2};
* no EXIF orientation other than 1 (imdecode would rotate).
Anything else raises `Unsupported`.  A damaged header, corrupt entropy data (an invalid code, data that ends before the last
MCU, a wrong RST sequence or count) and dequantised coefficients past MAX_DEQUANT raise `Corrupt`: libjpeg warns and fills in
pixels there (or, past MAX_DEQUANT, gives pixels that depend on its build), the decoder refuses instead.  `parse` makes the
decoder's header checks in its order, with its messages.
"""
import numpy as np

# zig-zag index -> natural index, with libjpeg's 16 extra entries that send a run past 63 to 63
NATURAL = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63] + [63] * 16, np.int64)


class Unsupported(Exception):
    pass


class Corrupt(Exception):
    pass


class Huffman:
    """Canonical code of one DHT table: lookup over 16 bits of look-ahead -> (length, symbol); length 0 = no such code."""

    def __init__(self, counts, symbols, is_dc):
        if sum(counts) > 256 or sum(counts) != len(symbols):
            raise Corrupt("bad Huffman table")
        self.counts, self.symbols = list(counts), list(symbols)
        self.length = np.zeros(1 << 16, np.int64)
        self.symbol = np.zeros(1 << 16, np.int64)
        code, k = 0, 0
        for l in range(1, 17):
            for _ in range(counts[l - 1]):
                lo, hi = code << (16 - l), (code + 1) << (16 - l)
                self.length[lo:hi] = l
                self.symbol[lo:hi] = symbols[k]
                code += 1
                k += 1
            if counts[l - 1] and code >= (1 << l):  # jpeg_make_d_derived_tbl: no code may be all ones
                raise Corrupt("bad Huffman table")
            code <<= 1
        if is_dc and any(s > 15 for s in symbols):
            raise Corrupt("bad Huffman table")


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def _exif_orientation(p):
    """Orientation tag (0x0112) of IFD0 of an APP1 Exif payload, or 1."""
    if len(p) < 14 or p[:6] != b"Exif\x00\x00":
        return 1
    t = p[6:]
    if t[:2] == b"II":
        rd = lambda o, n: int.from_bytes(t[o:o + n], "little")  # noqa: E731
    elif t[:2] == b"MM":
        rd = lambda o, n: int.from_bytes(t[o:o + n], "big")  # noqa: E731
    else:
        return 1
    ifd = rd(4, 4)
    if ifd + 2 > len(t):
        return 1
    for e in range(rd(ifd, 2)):
        o = ifd + 2 + 12 * e
        if o + 12 > len(t):
            break
        if rd(o, 2) == 0x0112:
            return rd(o + 8, 2)
    return 1


SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "differential sequential", 0xC6: "differential progressive",
             0xC7: "differential lossless", 0xC9: "arithmetic-coded", 0xCA: "arithmetic-coded progressive",
             0xCB: "arithmetic-coded lossless", 0xCD: "arithmetic-coded differential", 0xCE: "arithmetic-coded differential",
             0xCF: "arithmetic-coded differential"}


def parse(buf):
    """Markers up to the start of the entropy-coded data, checked in the decoder's order with its messages.  Returns a dict
    describing the frame and its one scan."""
    b = bytes(buf)
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise Corrupt("not a JPEG file (no SOI marker)")
    q = [None] * 4
    dc, ac = [None] * 4, [None] * 4
    ri, jfif, adobe, orient, sof = 0, False, None, 1, None
    i = 2
    while True:
        if i < len(b) and b[i] != 0xFF:
            raise Corrupt("garbage between markers")
        while i < len(b) and b[i] == 0xFF:
            i += 1
        if i + 2 >= len(b):
            raise Corrupt("file ends before the scan")
        m = b[i]
        i += 1
        if m == 0xD8 or m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise Corrupt("unexpected marker before the scan")
        L = _u16(b, i)
        if L < 2 or i + L > len(b):
            raise Corrupt("marker segment runs past the end of the file")
        p = b[i + 2:i + L]
        i += L
        if m in SOF_NAMES:
            raise Unsupported("%s JPEG (SOF%d) is not supported" % (SOF_NAMES[m], m - 0xC0))
        if m in (0xC0, 0xC1):
            if len(p) < 6:
                raise Corrupt("short frame header")
            prec, h, w, nf = p[0], _u16(p, 1), _u16(p, 3), p[5]
            if prec != 8:
                raise Unsupported("%d-bit samples are not supported (8-bit only)" % prec)
            if nf == 4:
                raise Unsupported("CMYK / 4-component JPEG is not supported")
            if nf not in (1, 3):
                raise Unsupported("%d-component JPEG is not supported" % nf)
            if len(p) < 6 + 3 * nf:
                raise Corrupt("short frame header")
            comps = [dict(id=p[6 + 3 * k], h=p[7 + 3 * k] >> 4, v=p[7 + 3 * k] & 15, tq=p[8 + 3 * k]) for k in range(nf)]
            sof = dict(w=w, h=h, comps=comps)
        elif m == 0xC4:
            o = 0
            while o < len(p):
                if o + 17 > len(p):
                    raise Corrupt("short DHT segment")
                tc, th = p[o] >> 4, p[o] & 15
                if th > 3 or tc > 1:
                    raise Corrupt("bad DHT table id")
                counts = list(p[o + 1:o + 17])
                syms = list(p[o + 17:o + 17 + sum(counts)])
                (dc if tc == 0 else ac)[th] = Huffman(counts, syms, tc == 0)
                o += 17 + sum(counts)
        elif m == 0xDB:
            o = 0
            while o < len(p):
                pq, tq = p[o] >> 4, p[o] & 15
                if tq > 3:
                    raise Corrupt("bad DQT table id")
                n = 2 if pq else 1
                if o + 1 + 64 * n > len(p):
                    raise Corrupt("short DQT segment")
                vals = [(_u16(p, o + 1 + 2 * k) if pq else p[o + 1 + k]) for k in range(64)]
                nat = np.zeros(64, np.int64)
                nat[NATURAL[:64]] = vals
                q[tq] = nat
                o += 1 + 64 * n
        elif m == 0xDD:
            if len(p) < 2:
                raise Corrupt("short DRI segment")
            ri = _u16(p, 0)
        elif m == 0xE0:
            jfif = jfif or p[:5] == b"JFIF\x00"
        elif m == 0xE1:
            o = _exif_orientation(p)
            orient = o if orient == 1 else orient
        elif m == 0xEE:
            if p[:5] == b"Adobe" and len(p) >= 12:
                adobe = p[11]
        elif m == 0xDA:
            if sof is None:
                raise Corrupt("scan before the frame header")
            if len(p) < 1 or len(p) < 4 + 2 * p[0]:
                raise Corrupt("short scan header")
            ns = p[0]
            scomps = [(p[1 + 2 * k], p[2 + 2 * k] >> 4, p[2 + 2 * k] & 15) for k in range(ns)]
            ss, se, ahal = p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns]
            return _validate(sof, scomps, (ss, se, ahal), q, dc, ac, ri, jfif, adobe, orient, i, b)


def _validate(sof, scomps, spectral, q, dc, ac, ri, jfif, adobe, orient, data_off, b):
    comps, nf = sof["comps"], len(sof["comps"])
    if sof["w"] == 0 or sof["h"] == 0:
        raise Unsupported("JPEG without its size in the frame header (DNL) is not supported")
    if len(scomps) != nf:
        raise Unsupported("multi-scan JPEG is not supported (the first scan holds %d of %d components)" % (len(scomps), nf))
    if spectral != (0, 63, 0):
        raise Corrupt("bad spectral selection in a sequential scan")
    if nf == 3:
        ids = [c["id"] for c in comps]
        ycc = jfif or (adobe == 1 if adobe is not None else ids == [1, 2, 3])
        if not ycc:
            raise Unsupported("RGB-coded JPEG is not supported (YCbCr only)")
        if any(c["h"] != 1 or c["v"] != 1 for c in comps[1:]) or comps[0]["h"] not in (1, 2) or comps[0]["v"] not in (1, 2):
            raise Unsupported("chroma subsampling %s is not supported (4:4:4, 4:2:2, 4:4:0, 4:2:0 only)" %
                              ",".join("%dx%d" % (c["h"], c["v"]) for c in comps))
    if orient in range(2, 9):
        raise Unsupported("EXIF orientation %d is not supported (imdecode would rotate the image)" % orient)
    out = []
    for cid, td, ta in scomps:
        match = [c for c in comps if c["id"] == cid]
        if not match or td > 3 or ta > 3:
            raise Corrupt("scan component does not match the frame")
        c = dict(match[-1])
        if q[c["tq"] & 3] is None or dc[td] is None or ac[ta] is None:
            raise Corrupt("scan uses an undefined table")
        c.update(q=q[c["tq"] & 3].copy(), dc=dc[td], ac=ac[ta])
        out.append(c)
    w, h = sof["w"], sof["h"]
    if nf == 1:
        hm = vm = 1
        out[0]["h"] = out[0]["v"] = 1  # a one-component scan is not interleaved: one block per MCU
    else:
        hm, vm = out[0]["h"], out[0]["v"]
        if any(c["h"] != 1 or c["v"] != 1 for c in out[1:]):
            raise Unsupported("a scan that does not start with the luma component is not supported")
    mx, my = -(-w // (8 * hm)), -(-h // (8 * vm))
    return dict(w=w, h=h, comps=out, hmax=hm, vmax=vm, mcux=mx, mcuy=my, ri=ri, data_off=data_off, buf=b)


def _segments(hd):
    """The entropy-coded data cut at its RST markers, stuffed zeros removed.  Returns the list of segments (bytes) and
    whether a marker other than RSTn ends the data (EOI; imdecode refuses a file without one)."""
    b, i = hd["buf"], hd["data_off"]
    segs, cur, expect, ended = [], bytearray(), 0, False
    n_mcu = hd["mcux"] * hd["mcuy"]
    nseg = -(-n_mcu // hd["ri"]) if hd["ri"] else 1
    while i < len(b):
        c = b[i]
        if c != 0xFF:
            cur.append(c)
            i += 1
            continue
        j = i + 1
        while j < len(b) and b[j] == 0xFF:
            j += 1
        if j >= len(b):
            break
        if b[j] == 0x00:
            cur.append(0xFF)
            i = j + 1
            continue
        if 0xD0 <= b[j] <= 0xD7:
            if b[j] != 0xD0 + (expect & 7):
                raise Corrupt("wrong RST marker sequence (RST%d where RST%d is due)" % (b[j] - 0xD0, expect & 7))
            expect += 1
            segs.append(bytes(cur))
            cur = bytearray()
            i = j + 1
            continue
        ended = True
        break
    segs.append(bytes(cur))
    if len(segs) != nseg:
        raise Corrupt("%d restart intervals where %d are due" % (len(segs), nseg))
    return segs, ended


def blocks_per_mcu(hd):
    return sum(c["h"] * c["v"] for c in hd["comps"])


def mcu_layout(hd):
    """For each block of an MCU: (component, x offset, y offset) in blocks."""
    return [(ci, bx, by) for ci, c in enumerate(hd["comps"]) for by in range(c["v"]) for bx in range(c["h"])]


def coefficients(hd):
    """Entropy decode.  Returns int64 [n_blocks, 64] in decode (MCU) order, natural order, absolute DC.

    Each restart interval is decoded on its own, up to its first error.  A code whose 16-bit look-ahead reaches past the
    interval's end and matches no code counts as the interval ending early (what follows the end is not the interval's
    data).  When intervals fail, an invalid code in any of them is the file's error, else the interval that ends early."""
    segs, ended = _segments(hd)
    lay = mcu_layout(hd)
    bpm = len(lay)
    n_mcu = hd["mcux"] * hd["mcuy"]
    ri = hd["ri"] or n_mcu
    out = np.zeros((n_mcu * bpm, 64), np.int64)
    errors = []
    for s, data in enumerate(segs):
        try:
            _decode_interval(hd, s, data, out, lay, ri, n_mcu)
        except Corrupt as e:
            errors.append(e)
    if errors:
        raise next((e for e in errors if "invalid Huffman code" in str(e)), errors[0])
    if not ended:
        raise Corrupt("entropy-coded data is not ended by a marker (truncated file)")
    out = ((out + 32768) & 0xFFFF) - 32768  # JCOEF is 16-bit
    return out


def _decode_interval(hd, s, data, out, lay, ri, n_mcu):
    bpm = len(lay)
    comps = hd["comps"]
    nbits = 8 * len(data)
    d = data + b"\x00" * 8
    pos = 0
    pred = [0] * len(comps)

    def peek(p, n):
        v = int.from_bytes(d[p >> 3:(p >> 3) + 5].ljust(5, b"\x00"), "big")
        return (v >> (40 - (p & 7) - n)) & ((1 << n) - 1)

    def short():
        return Corrupt("entropy-coded data ends before the last MCU of restart interval %d" % s)

    def decode(tab, p):
        k = peek(p, 16)
        l = int(tab.length[k])
        if l == 0:
            raise short() if p + 16 > nbits else Corrupt("invalid Huffman code in restart interval %d" % s)
        return int(tab.symbol[k]), p + l

    def extend(v, n):
        return v - (1 << n) + 1 if v < (1 << (n - 1)) else v

    for m in range(s * ri, min((s + 1) * ri, n_mcu)):
        for k, (ci, _, _) in enumerate(lay):
            c = comps[ci]
            blk = out[m * bpm + k]
            sym, pos = decode(c["dc"], pos)
            diff = 0
            if sym:
                diff = extend(peek(pos, sym), sym)
                pos += sym
            pred[ci] += diff
            blk[0] = pred[ci]
            z = 1
            while z < 64:
                sym, pos = decode(c["ac"], pos)
                r, n = sym >> 4, sym & 15
                if n:
                    z += r
                    blk[NATURAL[z]] = extend(peek(pos, n), n)
                    pos += n
                else:
                    if r != 15:
                        break
                    z += 15
                z += 1
            if pos > nbits:
                raise short()


# The largest |coefficient x quantisation value| jpeg_fdct_islow and libjpeg-turbo's quantiser produce from 8-bit samples at
# any 8- or 16-bit table entry (the DC of a flat block of 0 or 255 quantised by 2048; derived in test_jpeg_damage_cpu.py).
# Past it, the pixels imdecode gives depend on how libjpeg-turbo was built (a single coefficient past the bound already
# drives the C IDCT's output past the +-512 its range-limit table wraps at, where the SIMD IDCT differs), so the decoder
# refuses such a file as corrupt.
MAX_DEQUANT = 2048


def check_range(hd, coef):
    """Raises Corrupt if a dequantised coefficient (int16 coefficient times the int16 table entry) exceeds MAX_DEQUANT."""
    lay = mcu_layout(hd)
    for k, (ci, _, _) in enumerate(lay):
        qt16 = ((np.asarray(hd["comps"][ci]["q"], np.int64) + 32768) & 0xFFFF) - 32768
        if (np.abs(coef[k::len(lay)] * qt16) > MAX_DEQUANT).any():
            raise Corrupt("dequantised DCT coefficient or IDCT output out of range (corrupt data)")


# jpeg_idct_islow (jidctint.c), CONST_BITS 13, PASS1_BITS 2
F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
         f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(c0, c1, c2, c3, c4, c5, c6, c7):
    z1 = (c2 + c6) * F["f0541"]
    tmp2 = z1 - c6 * F["f1847"]
    tmp3 = z1 + c2 * F["f0765"]
    tmp0 = (c0 + c4) << 13
    tmp1 = (c0 - c4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = c7, c5, c3, c1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F["f1175"]
    o0 = o0 * F["f0298"]
    o1 = o1 * F["f2053"]
    o2 = o2 * F["f3072"]
    o3 = o3 * F["f1501"]
    z1 = z1 * -F["f0899"]
    z2 = z2 * -F["f2562"]
    z3 = z3 * -F["f1961"] + z5
    z4 = z4 * -F["f0390"] + z5
    o0 += z1 + z3
    o1 += z2 + z4
    o2 += z2 + z3
    o3 += z1 + z4
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def idct(coef, qt):
    """Dequantise and inverse-DCT blocks: coef int64 [n, 64] (natural order), qt [64] -> uint8 [n, 8, 8]."""
    qt16 = ((np.asarray(qt, np.int64) + 32768) & 0xFFFF) - 32768  # ISLOW_MULT_TYPE is 16-bit
    d = (coef * qt16).reshape(-1, 8, 8)
    cols = _idct_1d(*[d[:, k, :] for k in range(8)])  # pass 1 over columns: ws[row k][col]
    ws = np.stack([_descale(v, 13 - 2) for v in cols], 1)
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)])
    out = np.stack([_descale(v, 13 + 2 + 3) for v in rows], 2)
    if ((out < -512) | (out > 511)).any():  # the range-limit table wraps here, libjpeg-turbo's SIMD IDCT saturates
        raise Corrupt("dequantised DCT coefficient or IDCT output out of range (corrupt data)")
    # range_limit[x & RANGE_MASK] of the post-IDCT table: x taken as a signed 10-bit value, + 128, clamped
    s = ((out & 1023) ^ 512) - 512
    return np.clip(s + 128, 0, 255).astype(np.uint8)


def idct_planes(hd, coef):
    """Component planes padded to whole MCUs (uint8 [rows, cols] each)."""
    lay = mcu_layout(hd)
    bpm = len(lay)
    mx, my = hd["mcux"], hd["mcuy"]
    planes = []
    for ci, c in enumerate(hd["comps"]):
        P = np.zeros((my * c["v"] * 8, mx * c["h"] * 8), np.uint8)
        V = P.reshape(my, c["v"], 8, mx, c["h"], 8)  # (MCU row, block row, pixel row, MCU column, block column, pixel column)
        for k, (cj, bx, by) in enumerate(lay):
            if cj == ci:
                V[:, by, :, :, bx, :] = idct(coef[k::bpm], c["q"]).reshape(my, mx, 8, 8).transpose(0, 2, 1, 3)
        planes.append(P)
    return planes


def _up_h2(row_in, cw, fancy):
    """h2v1 upsampling of [..., cw] samples -> [..., 2 cw]"""
    x = row_in[..., :cw].astype(np.int64)
    out = np.empty(x.shape[:-1] + (2 * cw,), np.int64)
    if not fancy:
        out[..., 0::2] = x
        out[..., 1::2] = x
        return out
    left = np.concatenate([x[..., :1], x[..., :-1]], -1)
    right = np.concatenate([x[..., 1:], x[..., -1:]], -1)
    out[..., 0::2] = (3 * x + left + 1) >> 2
    out[..., 1::2] = (3 * x + right + 2) >> 2
    out[..., 0] = x[..., 0]
    out[..., -1] = x[..., -1]
    return out


def _upsample(hd, P, ci):
    """Chroma plane -> full-size plane (int64 [h, w]) by libjpeg's upsampler for this sampling."""
    w, h, hm, vm = hd["w"], hd["h"], hd["hmax"], hd["vmax"]
    c = hd["comps"][ci]
    cw, ch = -(-w * c["h"] // hm), -(-h * c["v"] // vm)
    x = P[:ch, :cw].astype(np.int64)
    fh, fv = hm // c["h"], vm // c["v"]
    if fh == 1 and fv == 1:
        return x
    if fv == 1:  # h2v1
        return _up_h2(x, cw, cw > 2)[:, :w]
    up = np.concatenate([x[:1], x[:-1]], 0)
    dn = np.concatenate([x[1:], x[-1:]], 0)
    rows = np.empty((2 * ch, cw), np.int64)
    if fh == 1:  # h1v2: always the triangle filter
        rows[0::2] = (3 * x + up + 1) >> 2
        rows[1::2] = (3 * x + dn + 2) >> 2
        return rows[:h]
    if cw <= 2:  # h2v2 box
        return np.repeat(np.repeat(x, 2, 0), 2, 1)[:h, :w]
    cs = np.empty((2 * ch, cw), np.int64)
    cs[0::2] = 3 * x + up
    cs[1::2] = 3 * x + dn
    left = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
    right = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * cs + left + 8) >> 4
    out[:, 1::2] = (3 * cs + right + 7) >> 4
    out[:, 0] = (cs[:, 0] * 4 + 8) >> 4
    out[:, -1] = (cs[:, -1] * 4 + 7) >> 4
    return out[:h, :w]


def to_bgr(hd, planes):
    """Upsampling and ycc_rgb_convert (jdcolor.c, SCALEBITS 16) -> uint8 [h, w, 3] BGR."""
    w, h = hd["w"], hd["h"]
    y = planes[0][:h, :w].astype(np.int64)
    if len(planes) == 1:
        return np.repeat(y[:, :, None], 3, 2).astype(np.uint8)
    cb = _upsample(hd, planes[1], 1) - 128
    cr = _upsample(hd, planes[2], 2) - 128
    half = 1 << 15
    r = y + ((91881 * cr + half) >> 16)
    g = y + ((-46802 * cr + (-22554 * cb + half)) >> 16)
    b = y + ((116130 * cb + half) >> 16)
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def bgr_to_gray(bgr):
    """cvtColor(COLOR_BGR2GRAY) on uint8: (B*3735 + G*19235 + R*9798 + 2^14) >> 15"""
    x = bgr.astype(np.int64)
    return ((x[..., 0] * 3735 + x[..., 1] * 19235 + x[..., 2] * 9798 + 16384) >> 15).astype(np.uint8)


def decode(buf, channels=3):
    hd = parse(buf)
    coef = coefficients(hd)
    check_range(hd, coef)
    bgr = to_bgr(hd, idct_planes(hd, coef))
    return bgr if channels == 3 else bgr_to_gray(bgr)
