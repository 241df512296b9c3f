"""A numpy restatement of `cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q])` (libjpeg-turbo's compressor with OpenCV's
defaults: baseline, standard Huffman tables, islow DCT, no restart markers) for the two configurations the project writes:
one gray component (the flow planes) and YCbCr 4:2:0 from BGR (the `-s=0` frames).  Test infrastructure, pinned live
against cv2 in tests/test_jpeg_encode_cpu.py; the CUDA encoder (denseflow_b200/csrc/jpeg_encode.cu) is checked against it.

Edge padding, as the byte pin confirms it:
* gray and luma: the last column and the last row are replicated up to whole blocks (expand_right_edge, jcsample.c;
  expand_bottom_edge, jcprepct.c);
* 4:2:0 luma blocks outside the component's width_in_blocks / height_in_blocks but inside an MCU are dummy blocks
  (compress_data, jccoefct.c): AC zero, DC copied from the block to the left, or in the bottom MCU row from the last block
  of the MCU's row above (Y01 for both Y10 and Y11);
* 4:2:0 chroma columns past ceil(w / 2) are downsampled from full-resolution columns replicated to twice the padded
  chroma width, so they keep the alternating 1 / 2 bias;
* 4:2:0 chroma rows past ceil(h / 2) replicate the last *downsampled* row (pre_process_data pads the full-resolution rows
  only to the row group, then the downsampled rows to the iMCU height).
"""
import numpy as np

import ycc_restate as Y
from jpeg_restate import NATURAL

ZIGZAG = NATURAL[:64]  # zig-zag index -> natural index

# JPEG Annex K.1, natural order
STD_LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_Q = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, np.int64)

# JPEG Annex K.3: (bits[1..16], values) of the DC / AC tables, luminance then chrominance
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
    0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
    0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
    0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])


def quant_table(basic, quality):
    """jpeg_set_quality -> jpeg_quality_scaling + jpeg_add_quant_table(force_baseline=TRUE), natural order"""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((basic * scale + 50) // 100, 1, 255)


def reciprocal(divisor):
    """compute_reciprocal (jcdctmgr.c) with 16-bit DCTELEM: (reciprocal, correction, total shift r)"""
    b = int(divisor).bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, divisor)
    c = divisor // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= divisor // 2:
        c += 1
    else:
        fq += 1
    return fq, c, r


def quantize(coef, qtab):
    """libjpeg-turbo's quantize (jcdctmgr.c) as written: |x| + correction, times the reciprocal, shifted; coef int64 [..., 64]
    natural order, qtab natural order.  The divisor is quantval << 3 (the islow DCT's output is scaled by 8)."""
    rc = np.array([reciprocal(int(d) << 3) for d in qtab], np.int64)
    a = np.abs(coef)
    q = ((a + rc[:, 1]) * rc[:, 0]) >> rc[:, 2]
    return np.where(coef < 0, -q, q)


# jpeg_fdct_islow (jfdctint.c), CONST_BITS 13, PASS1_BITS 2
def _fdct_1d(d, pass1):
    s = [d[..., k] for k in range(8)]
    tmp0, tmp7 = s[0] + s[7], s[0] - s[7]
    tmp1, tmp6 = s[1] + s[6], s[1] - s[6]
    tmp2, tmp5 = s[2] + s[5], s[2] - s[5]
    tmp3, tmp4 = s[3] + s[4], s[3] - s[4]
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    n = 13 - 2 if pass1 else 13 + 2

    def ds(x, k):
        return (x + (1 << (k - 1))) >> k

    o = [None] * 8
    if pass1:
        o[0], o[4] = (tmp10 + tmp11) << 2, (tmp10 - tmp11) << 2
    else:
        o[0], o[4] = ds(tmp10 + tmp11, 2), ds(tmp10 - tmp11, 2)
    z1 = (tmp12 + tmp13) * 4433
    o[2] = ds(z1 + tmp13 * 6270, n)
    o[6] = ds(z1 - tmp12 * 15137, n)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * 9633
    tmp4, tmp5, tmp6, tmp7 = tmp4 * 2446, tmp5 * 16819, tmp6 * 25172, tmp7 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    o[7] = ds(tmp4 + z1 + z3, n)
    o[5] = ds(tmp5 + z2 + z4, n)
    o[3] = ds(tmp6 + z2 + z3, n)
    o[1] = ds(tmp7 + z1 + z4, n)
    return np.stack(o, -1)


def fdct(blocks):
    """uint8 [n, 8, 8] -> int64 [n, 64] natural order (scaled by 8, as libjpeg's islow DCT leaves it)"""
    x = blocks.astype(np.int64) - 128
    x = _fdct_1d(x, True)                                      # rows
    x = _fdct_1d(x.transpose(0, 2, 1), False).transpose(0, 2, 1)  # columns
    return x.reshape(-1, 64)


def _blocks(plane):
    """[8 H, 8 W] -> [H * W, 8, 8] in raster order"""
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


def _pad_edge(p, rows, cols):
    return np.pad(p, ((0, rows - p.shape[0]), (0, cols - p.shape[1])), mode="edge")


def chroma_padded(c_full, w, h):
    """Chroma plane of the 4:2:0 encode padded to 8 * ceil(w / 16) columns and 8 * ceil(h / 16) rows (see the module notes)"""
    cw, ch = 8 * -(-w // 16), 8 * -(-h // 16)
    full = np.pad(c_full, ((0, h & 1), (0, 2 * cw - w)), mode="edge").astype(np.int64)
    s = full[0::2, 0::2] + full[0::2, 1::2] + full[1::2, 0::2] + full[1::2, 1::2]
    d = ((s + (1 + (np.arange(cw) & 1))[None, :]) >> 2).astype(np.uint8)
    return _pad_edge(d, ch, cw)


def coefficients(img, quality=95):
    """Quantised coefficients in encode (MCU) order, natural order: int64 [n_blocks, 64], and the component of each block."""
    if img.ndim == 2:
        h, w = img.shape
        wb, hb = -(-w // 8), -(-h // 8)
        p = _pad_edge(img, 8 * hb, 8 * wb)
        return quantize(fdct(_blocks(p)), quant_table(STD_LUMA_Q, quality)), np.zeros(wb * hb, np.int64)
    h, w = img.shape[:2]
    yy, cb, cr = Y.bgr_to_ycc(img)
    mx, my = -(-w // 16), -(-h // 16)
    wb, hb = -(-w // 8), -(-h // 8)
    ly = quantize(fdct(_blocks(_pad_edge(yy.astype(np.uint8), 8 * hb, 8 * wb))), quant_table(STD_LUMA_Q, quality))
    ly = ly.reshape(hb, wb, 64)
    qc = quant_table(STD_CHROMA_Q, quality)
    lcb = quantize(fdct(_blocks(chroma_padded(cb, w, h))), qc).reshape(my, mx, 64)
    lcr = quantize(fdct(_blocks(chroma_padded(cr, w, h))), qc).reshape(my, mx, 64)
    out = np.zeros((my, mx, 6, 64), np.int64)
    for k in range(4):
        bx, by = k & 1, k >> 1
        sub = ly[by::2, bx::2]
        out[:sub.shape[0], :sub.shape[1], k] = sub
    # dummy luma blocks (compress_data): right edge takes the DC of the block to its left, the bottom MCU row's missing
    # block row takes the DC of the last block of the row above
    if wb & 1:
        out[:, -1, 1, 0] = out[:, -1, 0, 0]
        out[:, -1, 3, 0] = out[:, -1, 2, 0]
    if hb & 1:
        out[-1, :, 2, 0] = out[-1, :, 1, 0]
        out[-1, :, 3, 0] = out[-1, :, 1, 0]
    out[:, :, 4] = lcb
    out[:, :, 5] = lcr
    return out.reshape(-1, 64), np.tile([0, 0, 0, 0, 1, 2], mx * my)


def _derive(table):
    """jpeg_make_c_derived_tbl: symbol -> (code, length)"""
    bits, vals = table
    code, k, out = 0, 0, {}
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


def _dht(tc, th, table):
    bits, vals = table
    body = bytes([tc << 4 | th]) + bytes(bits) + bytes(vals)
    return b"\xff\xc4" + (len(body) + 2).to_bytes(2, "big") + body


def header(w, h, components, quality=95):
    """SOI, JFIF APP0, DQT(s), SOF0, DHT(s), SOS: every byte before the entropy-coded data"""
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    tabs = [quant_table(STD_LUMA_Q, quality)] + ([quant_table(STD_CHROMA_Q, quality)] if components == 3 else [])
    for i, t in enumerate(tabs):
        out += b"\xff\xdb\x00\x43" + bytes([i]) + bytes(int(v) for v in t[ZIGZAG])
    out += b"\xff\xc0" + (8 + 3 * components).to_bytes(2, "big") + b"\x08" + h.to_bytes(2, "big") + w.to_bytes(2, "big")
    out += bytes([components])
    if components == 1:
        out += b"\x01\x11\x00"
    else:
        out += b"\x01\x22\x00\x02\x11\x01\x03\x11\x01"
    out += _dht(0, 0, DC_LUMA) + _dht(1, 0, AC_LUMA)
    if components == 3:
        out += _dht(0, 1, DC_CHROMA) + _dht(1, 1, AC_CHROMA)
    out += b"\xff\xda" + (6 + 2 * components).to_bytes(2, "big") + bytes([components])
    out += b"\x01\x00" if components == 1 else b"\x01\x00\x02\x11\x03\x11"
    out += b"\x00\x3f\x00"
    return bytes(out)


def _category(v):
    return int(abs(int(v))).bit_length()


def entropy(coef, comp, with_bits=False):
    """Huffman-code the blocks (encode_one_block, jchuff.c), flush with 1-bits, stuff a 0x00 after every 0xFF.  with_bits:
    also return the number of coded bits before the flush."""
    tabs = [(_derive(DC_LUMA), _derive(AC_LUMA)), (_derive(DC_CHROMA), _derive(AC_CHROMA))]
    bits = []  # (value, length) pairs
    pred = [0, 0, 0]
    zz = coef[:, ZIGZAG]
    for blk, c in zip(zz.tolist(), comp.tolist()):
        dct, act = tabs[min(c, 1)]
        diff = blk[0] - pred[c]
        pred[c] = blk[0]
        n = _category(diff)
        bits.append(dct[n])
        if n:
            bits.append(((diff if diff >= 0 else diff - 1) & ((1 << n) - 1), n))
        r = 0
        for k in range(1, 64):
            v = blk[k]
            if v == 0:
                r += 1
                continue
            while r > 15:
                bits.append(act[0xF0])
                r -= 16
            n = _category(v)
            bits.append(act[(r << 4) | n])
            bits.append(((v if v >= 0 else v - 1) & ((1 << n) - 1), n))
            r = 0
        if r:
            bits.append(act[0x00])
    acc, nacc = 0, 0
    out = bytearray()
    for v, l in bits:
        acc = (acc << l) | v
        nacc += l
        while nacc >= 8:
            out.append((acc >> (nacc - 8)) & 0xFF)
            nacc -= 8
        acc &= (1 << nacc) - 1
    nbits = 8 * len(out) + nacc
    if nacc:
        out.append(((acc << (8 - nacc)) | ((1 << (8 - nacc)) - 1)) & 0xFF)
    data = bytes(out).replace(b"\xff", b"\xff\x00")
    return (data, nbits) if with_bits else data


def encode(img, quality=95):
    """imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, quality]) for a uint8 [h, w] gray or [h, w, 3] BGR image"""
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    coef, comp = coefficients(img, quality)
    return header(w, h, 1 if img.ndim == 2 else 3, quality) + entropy(coef, comp) + b"\xff\xd9"


def locate(got, want):
    """A readable account of the first difference between two JPEG files: the first block and coefficient whose decoded
    values differ (the DCT, quantiser or padding), else the first differing byte (the header or the entropy coder)."""
    import jpeg_restate as J
    got, want = bytes(got), bytes(want)
    if got == want:
        return "identical"
    try:
        cg, cw = J.coefficients(J.parse(got)), J.coefficients(J.parse(want))
    except Exception as e:  # noqa: BLE001 - a file that does not decode is reported as such
        cg = cw = None
        why = "a file does not decode (%s)" % e
    if cg is not None:
        if cg.shape != cw.shape:
            why = "block counts differ (%d vs %d)" % (len(cg), len(cw))
        else:
            d = np.argwhere(cg != cw)
            if len(d):
                b, k = d[0]
                return "block %d (MCU order), coefficient %d (natural order): %d vs %d" % (b, k, cg[b, k], cw[b, k])
            why = "coefficients equal"
    n = min(len(got), len(want))
    i = next((i for i in range(n) if got[i] != want[i]), n)
    return "%s; first differing byte %d of %d / %d" % (why, i, len(got), len(want))
