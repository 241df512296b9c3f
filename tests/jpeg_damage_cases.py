"""Damaged and hand-built JPEG files for the decoder's refusals, in the style of deflate_cases.py: each case is a name, the
file's bytes and the edge it is built to reach, and the builder asserts that the case reaches it.  Expected verdicts come
from the restatement (jpeg_restate.verdict), never from hand-written lists.

* `write` is a small baseline writer: given quantisation tables, int16 blocks per MCU (or explicit Huffman symbols per
  block) and a restart interval, it writes the bytes, so files can hold what no encoder writes (runs past zig-zag index 63,
  absolute DC beyond int16, dequantised values past what an 8-bit encoder produces).
* `entropy_cases` damages the scan of small cv2 files of every sampling, with and without restart intervals.
* `header_cases` damages one marker segment at a time.
* `coefficient_cases` holds the hand-built files.
"""
import numpy as np

import jpeg_cases as J
import jpeg_restate as R

ZIGZAG = R.NATURAL[:64]
_HV = {"gray": [(1, 1)], "444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "440": [(1, 2), (1, 1), (1, 1)],
       "420": [(2, 2), (1, 1), (1, 1)]}

# Huffman tables that code every DC category 0..15 (5-bit codes) and every AC symbol (8-bit codes); neither is complete
DC_ALL = ([0, 0, 0, 0, 16] + [0] * 11, list(range(16)))
AC_ALL = ([0] * 7 + [242] + [0] * 8, [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)])


def _codes(table):
    bits, vals = table
    code, k, out = 0, 0, {}
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


def tokens(zz_block, pred):
    """Huffman symbols of one block (encode_one_block): ('dc', diff), ('ac', run, value), ('zrl',), ('eob',).  zz_block: 64
    coefficients in zig-zag order with absolute DC."""
    out = [("dc", int(zz_block[0]) - pred)]
    r = 0
    for k in range(1, 64):
        v = int(zz_block[k])
        if v == 0:
            r += 1
            continue
        while r > 15:
            out.append(("zrl",))
            r -= 16
        out.append(("ac", r, v))
        r = 0
    if r:
        out.append(("eob",))
    return out


def _bits(v, n):
    return (v if v >= 0 else v - 1) & ((1 << n) - 1)


def write(w, h, sampling, blocks, q=None, qbits=8, ri=0, tables=(DC_ALL, AC_ALL)):
    """A baseline file of w x h and the given sampling.  blocks: int [n_blocks, 64] natural order with absolute DC, in MCU
    order (the restatement's `coefficients` layout), or a list of token lists per block (see `tokens`; DC differences).
    q: natural-order table used by every component (default all ones); qbits 8 or 16.  ri: restart interval in MCUs."""
    hv = _HV[sampling]
    nc = len(hv)
    q = np.ones(64, np.int64) if q is None else np.asarray(q, np.int64)
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    body = bytes([(1 if qbits == 16 else 0) << 4]) + b"".join(int(v).to_bytes(qbits // 8, "big") for v in q[ZIGZAG])
    out += b"\xff\xdb" + (len(body) + 2).to_bytes(2, "big") + body
    out += b"\xff\xc0" + (8 + 3 * nc).to_bytes(2, "big") + b"\x08" + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc])
    for c in range(nc):
        out += bytes([c + 1, hv[c][0] << 4 | hv[c][1], 0])
    for tc, t in ((0, tables[0]), (1, tables[1])):
        body = bytes([tc << 4]) + bytes(t[0]) + bytes(t[1])
        out += b"\xff\xc4" + (len(body) + 2).to_bytes(2, "big") + body
    if ri:
        out += b"\xff\xdd\x00\x04" + ri.to_bytes(2, "big")
    out += b"\xff\xda" + (6 + 2 * nc).to_bytes(2, "big") + bytes([nc]) + b"".join(bytes([c + 1, 0]) for c in range(nc))
    out += b"\x00\x3f\x00"
    lay = [c for c, (ch, cv) in enumerate(hv) for _ in range(ch * cv)] if nc > 1 else [0]
    bpm = len(lay)
    mcux, mcuy = -(-w // (8 * hv[0][0] if nc > 1 else 8)), -(-h // (8 * hv[0][1] if nc > 1 else 8))
    n_mcu = mcux * mcuy
    assert len(blocks) == n_mcu * bpm, (len(blocks), n_mcu * bpm)
    dc, ac = _codes(tables[0]), _codes(tables[1])
    out += _scan(blocks, lay, n_mcu, ri, dc, ac)
    return bytes(out) + b"\xff\xd9"


def _scan(blocks, lay, n_mcu, ri, dc, ac):
    bpm = len(lay)
    data = bytearray()
    seg = []
    pred = [0, 0, 0]
    for m in range(n_mcu):
        if ri and m and m % ri == 0:
            data += _flush(seg) + bytes([0xFF, 0xD0 + (m // ri - 1) % 8])
            seg, pred = [], [0, 0, 0]
        for k in range(bpm):
            b = blocks[m * bpm + k]
            c = lay[k]
            if isinstance(b, list):
                toks = b
            else:
                zz = np.asarray(b, np.int64)[ZIGZAG]
                toks = tokens(zz, pred[c])
                pred[c] = int(zz[0])
            for t in toks:
                if t[0] == "dc":
                    n = abs(t[1]).bit_length()
                    seg.append(dc[n])
                    if n:
                        seg.append((_bits(t[1], n), n))
                elif t[0] == "ac":
                    n = abs(t[2]).bit_length()
                    seg.append(ac[(t[1] << 4) | n])
                    seg.append((_bits(t[2], n), n))
                else:
                    seg.append(ac[0xF0 if t[0] == "zrl" else 0x00])
    return bytes(data + _flush(seg))


def _flush(codes):
    """Pack (value, length) codes, pad the last byte with 1-bits, stuff a 0x00 after every 0xFF."""
    acc, n = 0, 0
    for v, l in codes:
        acc, n = (acc << l) | v, n + l
    pad = -n % 8
    acc, n = (acc << pad) | ((1 << pad) - 1), n + pad
    return acc.to_bytes(n // 8, "big").replace(b"\xff", b"\xff\x00") if n else b""


# ---- verdicts ----------------------------------------------------------------------------------------------------------

ENTROPY_KINDS = (("RST marker sequence", "rst"), ("restart intervals where", "rst_count"), ("number of RST markers", "rst_count"),
                 ("invalid Huffman code", "code"), ("ends before the last MCU", "short"), ("not ended by a marker", "no_end"),
                 ("out of range", "range"))


def kind(message):
    """The kind of a refusal message (restatement's or decoder's): an entropy kind, or the header message itself."""
    m = message.split(": ", 1)[1] if message.startswith("frame ") else message
    return next((k for frag, k in ENTROPY_KINDS if frag in m), m)


def verdict(b):
    """('ok', None), ('corrupt', kind) or ('unsupported', message) by the restatement."""
    try:
        R.decode(b)
    except R.Unsupported as e:
        return "unsupported", kind(str(e))
    except R.Corrupt as e:
        return "corrupt", kind(str(e))
    return "ok", None


def scan_span(b):
    """(first byte of the entropy-coded data, index of the marker that ends the scan)"""
    i = R.parse(b)["data_off"]
    j = i
    while j + 1 < len(b):
        if b[j] == 0xFF and b[j + 1] not in (0x00, 0xFF) and not 0xD0 <= b[j + 1] <= 0xD7:
            return i, j
        j += 1
    return i, len(b)


def rst_positions(b):
    i, e = scan_span(b)
    return [j for j in range(i, e - 1) if b[j] == 0xFF and 0xD0 <= b[j + 1] <= 0xD7]


# ---- entropy damage ----------------------------------------------------------------------------------------------------

def _base_files():
    """name -> bytes: small cv2 files of every sampling, without restarts and with restart intervals 1 and 3"""
    out = {}
    for samp in J.SAMPLINGS:
        for ri in (0, 1, 3):
            out["%s_ri%d" % (samp, ri)] = J.encode(J.image("smooth" if ri else "noise", 24, 32), samp, 90, restart=ri)
    return out


def _flip(b, j, bit):
    x = bytearray(b)
    x[j] ^= 1 << bit
    return bytes(x)


def entropy_cases():
    """name -> (bytes, edge).  Edges: 'bitflip', 'marker', 'truncate', 'rst', 'junk', 'fill', 'no_eoi', 'order'.  A bit flip
    in a window (the first 32 scan bytes and 16 around each of two RST markers) takes every byte once, bit j mod 8, and all 8
    bits of the first 4 bytes; the gray 16x16 scan takes every bit.  Truncation takes every offset of the gray 16x16 and
    4:2:0 interval-3 scans, every 5th offset elsewhere."""
    cases = {}
    for name, b in _base_files().items():
        i, e = scan_span(b)
        rsts = rst_positions(b)
        window = set(range(i, min(i + 32, e)))
        for r in rsts[:2]:
            window |= set(range(max(i, r - 8), min(e, r + 8)))
        for j in sorted(window):
            for bit in (range(8) if j < i + 4 else [j % 8]):
                cases["%s/flip@%d.%d" % (name, j - i, bit)] = (_flip(b, j, bit), "bitflip")
        mid = (i + e) // 2
        for mk in [0xD9, 0xC4] + list(range(0xD0, 0xD8)):
            cases["%s/marker%02X@mid" % (name, mk)] = (b[:mid] + bytes([0xFF, mk]) + b[mid + 1:], "marker")
        for j in range(i, e, 1 if name == "420_ri3" else 5):
            cases["%s/cut@%d" % (name, j - i)] = (b[:j], "truncate")
            cases["%s/cut@%d+eoi" % (name, j - i)] = (b[:j] + b"\xff\xd9", "truncate")
        cases["%s/no_eoi" % name] = (b[:e], "no_eoi")
        cases["%s/junk_before_eoi" % name] = (b[:e] + b"\x12\x34\x56" + b[e:], "junk")
        cases["%s/fill_before_eoi" % name] = (b[:e] + b"\xff" * 5 + b[e:], "fill")
        if rsts:
            r = rsts[len(rsts) // 2]
            cases["%s/rst_deleted" % name] = (b[:r] + b[r + 2:], "rst")
            cases["%s/rst_duplicated" % name] = (b[:r + 2] + b[r:], "rst")
            cases["%s/rst_renumbered" % name] = (b[:r + 1] + bytes([0xD0 + (b[r + 1] - 0xD0 + 3) % 8]) + b[r + 2:], "rst")
            cases["%s/junk_before_rst" % name] = (b[:r] + b"\x12\x34" + b[r:], "junk")
            cases["%s/fill_before_rst" % name] = (b[:r] + b"\xff" * 4 + b[r:], "fill")
    # every bit of one whole gray 16x16 scan
    g = J.encode(J.image("noise", 16, 16), "gray", 90)
    i, e = scan_span(g)
    for j in range(i, e):
        for bit in range(8):
            cases["gray16/flip@%d.%d" % (j - i, bit)] = (_flip(g, j, bit), "bitflip")
        cases["gray16/cut@%d" % (j - i)] = (g[:j], "truncate")
        cases["gray16/cut@%d+eoi" % (j - i)] = (g[:j] + b"\xff\xd9", "truncate")
    # an interval that ends early before an interval holding an invalid code: the invalid code is the file's error
    b = J.encode(J.image("noise", 40, 48), "gray", 90, restart=3)
    r = rst_positions(b)
    i, _ = scan_span(b)
    cases["gray_ri3/short_then_code"] = (b[:i + 2] + b[r[0]:r[0] + 2] + b"\xff\x00" * 8 + b[r[0] + 2:], "order")
    cases["gray_ri3/code_then_short"] = (b[:i] + b"\xff\x00" * 8 + b[i:r[0] + 2] + b[r[0] + 2:r[1] - 20] + b[r[1]:], "order")
    return cases


# ---- header damage -----------------------------------------------------------------------------------------------------

def _segment(b, marker, nth=0):
    """(start, end) of the nth segment with this marker code (start at the 0xFF)"""
    i, seen = 2, 0
    while True:
        m, L = b[i + 1], _u16(b, i + 2)
        if m == marker:
            if seen == nth:
                return i, i + 2 + L
            seen += 1
        if m == 0xDA:
            raise KeyError(marker)
        i += 2 + L


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def _replace(b, marker, body, nth=0):
    s, e = _segment(b, marker, nth)
    return b[:s] + bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body + b[e:]


def _body(b, marker, nth=0):
    s, e = _segment(b, marker, nth)
    return bytearray(b[s + 4:e])


def header_cases():
    """name -> bytes: one marker segment damaged at a time (the edge is the decoder's header message the name stands for)"""
    base = J.encode(J.image("smooth", 24, 32), "420", 90)
    gray = J.encode(J.image("smooth", 24, 32), "gray", 90)
    c = {}
    dht = _body(base, 0xC4)  # DC table 0
    x = bytearray(dht)
    x[1:17] = bytes([0] * 7 + [255, 255] + [0] * 7)
    c["dht_counts_past_256"] = _replace(base, 0xC4, bytes(x) + bytes(510))
    c["dht_complete_code"] = _replace(base, 0xC4, bytes([0x00, 2] + [0] * 15 + [0, 1]))  # two 1-bit codes: "1" is all ones
    c["dht_complete_code_len3"] = _replace(base, 0xC4, bytes([0x00, 0, 4] + [0] * 14 + [0, 1, 2, 3]))
    c["dht_dc_symbol_16"] = _replace(base, 0xC4, bytes([0x00, 0, 1] + [0] * 14 + [16]))
    c["dht_tc_2"] = _replace(base, 0xC4, bytes([0x20]) + bytes(dht[1:]))
    c["dht_th_4"] = _replace(base, 0xC4, bytes([0x04]) + bytes(dht[1:]))
    c["dht_short"] = _replace(base, 0xC4, bytes(dht[:10]))
    c["dht_symbols_past_segment"] = _replace(base, 0xC4, bytes(dht[:-1]))
    dqt = _body(gray, 0xDB)
    c["dqt_tq_4"] = _replace(gray, 0xDB, bytes([0x04]) + bytes(dqt[1:]))
    c["dqt_short"] = _replace(gray, 0xDB, bytes(dqt[:40]))
    for v in (0, 32768, 65535):
        c["dqt16_all_%d" % v] = _replace(gray, 0xDB, bytes([0x10]) + v.to_bytes(2, "big") * 64)
    sof = _body(base, 0xC0)
    c["sof_short"] = _replace(base, 0xC0, bytes(sof[:5]))
    c["sof_short_components"] = _replace(base, 0xC0, bytes(sof[:12]))
    for name, (o, v) in {"sof_width_0": (3, 0), "sof_height_0": (1, 0)}.items():
        x = bytearray(sof)
        x[o:o + 2] = v.to_bytes(2, "big")
        c[name] = _replace(base, 0xC0, bytes(x))
    x = bytearray(sof)
    x[5] = 2
    c["sof_2_components"] = _replace(base, 0xC0, bytes(x[:12]))
    x = bytearray(sof)
    x[5] = 4
    c["sof_4_components"] = _replace(base, 0xC0, bytes(x) + b"\x04\x11\x01")
    x = bytearray(sof)
    x[0] = 12
    c["sof_12_bit"] = _replace(base, 0xC0, bytes(x))
    sos = _body(base, 0xDA)
    for name, (o, v) in {"sos_undefined_dc_table": (4, 0x21), "sos_table_id_4": (4, 0x41), "sos_unknown_component": (1, 9),
                         "sos_ss_1": (7, 1), "sos_se_62": (8, 62), "sos_ahal": (9, 0x10)}.items():
        x = bytearray(sos)
        x[o] = v
        c[name] = _replace(base, 0xDA, bytes(x))
    c["sos_short"] = _replace(base, 0xDA, bytes(sos[:5]))
    x = bytearray(sos)
    x[0] = 2
    c["sos_two_of_three_components"] = _replace(base, 0xDA, bytes(x[:5]) + bytes(x[7:]))
    s, e = _segment(gray, 0xC0)
    c["segment_past_eof"] = gray[:s + 2] + b"\xff\xf0" + gray[s + 4:s + 20]
    c["garbage_between_markers"] = gray[:s] + b"\x00\x11" + gray[s:]
    c["no_soi"] = gray[2:]
    c["ends_before_scan"] = gray[:s]
    c["scan_before_frame"] = gray[:s] + gray[_segment(gray, 0xDA)[0]:]
    c["unexpected_rst_before_scan"] = gray[:s] + b"\xff\xd0" + gray[s:]
    s, e = _segment(gray, 0xDA)
    c["dri_short"] = gray[:s] + b"\xff\xdd\x00\x03\x00" + gray[s:]
    c["dri_0"] = gray[:s] + b"\xff\xdd\x00\x04\x00\x00" + gray[s:]
    c["dri_past_mcu_count"] = gray[:s] + b"\xff\xdd\x00\x04\x01\x00" + gray[s:]
    c["progressive"] = J.encode(J.image("smooth", 24, 32), "420", 90, progressive=True)
    return c


# ---- hand-built files from coefficient blocks --------------------------------------------------------------------------

def coefficient_cases():
    """name -> (bytes, edge)"""
    c = {}
    q1 = np.ones(64, np.int64)
    # runs past zig-zag index 63: ZRL chains and a run/size symbol whose run ends past 63 (libjpeg writes index 63)
    c["zrl_past_63"] = (write(8, 8, "gray", [[("dc", 10), ("ac", 0, 3)] + [("zrl",)] * 4 + [("ac", 0, 5)]]), "run63")
    c["run_past_63"] = (write(8, 8, "gray", [[("dc", 10)] + [("zrl",)] * 3 + [("ac", 15, -7)]]), "run63")
    c["zrl_to_64"] = (write(16, 8, "gray", [[("dc", 10)] + [("zrl",)] * 4, [("dc", -4), ("ac", 2, 9), ("eob",)]]), "run63")
    c["eob_after_63"] = (write(16, 8, "gray", [[("dc", 1)] + [("ac", 0, 1)] * 63 + [("eob",)], [("dc", 1), ("eob",)]]), "eob63")
    # absolute DC past int16: the predictor wraps in the stored coefficient
    c["dc_wrap_up"] = (write(32, 8, "gray", [[("dc", 30000), ("eob",)], [("dc", 30000), ("eob",)], [("dc", -30000), ("eob",)],
                                             [("dc", -30000), ("eob",)]], q=np.zeros(64, np.int64)), "dc_wrap")
    c["dc_wrap_down_ri1"] = (write(32, 8, "gray", [[("dc", -32767), ("eob",)], [("dc", -32767), ("eob",)], [("dc", 5), ("eob",)],
                                                   [("dc", -20000), ("eob",)]], q=np.zeros(64, np.int64), ri=3), "dc_wrap")
    # dequantised values swept across the range encoders produce and past it, in DC and in each AC position class
    for k in (0, 1, 8, 9, 2, 18, 7, 63, 36):
        for v in (255, 1024, R.MAX_DEQUANT, R.MAX_DEQUANT + 1, 2176, 4095, 20000, 32767):
            for sign in (1, -1):
                blk = np.zeros((4, 64), np.int64)
                blk[1, k] = sign * v
                if k:
                    blk[2, k] = -sign * (v // 3)
                c["dq_k%d_%+d" % (k, sign * v)] = (write(16, 16, "gray", blk, q=q1, qbits=16), "dequant")
    for qv in (300, 4000, 40000):
        blk = np.zeros((4, 64), np.int64)
        blk[:, 0] = [7, -7, 2, 0]
        blk[:, 9] = [1, 0, -1, 0]
        c["dq_table_%d" % qv] = (write(16, 16, "gray", blk, q=np.full(64, qv), qbits=16), "dequant")
    return c


def all_cases():
    """name -> (bytes, edge) over the three builders"""
    out = dict(entropy_cases())
    out.update({"header/" + k: (v, "header") for k, v in header_cases().items()})
    out.update({"coef/" + k: v for k, v in coefficient_cases().items()})
    return out
