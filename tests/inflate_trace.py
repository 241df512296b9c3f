"""A small pure-Python inflate that keeps the structure of a deflate stream: per block its type, its code lengths and its
symbol list.  Tests use it to report the first block and symbol where two streams differ, and to pin the zlib rules the
GPU PNG encoder (denseflow_b200/csrc/png_encode.cu) restates."""
import zlib


class _Bits:
    def __init__(self, data, pos=0):
        self.d, self.i, self.buf, self.nb = data, pos, 0, 0

    def need(self, n):
        while self.nb < n:
            self.buf |= (self.d[self.i] if self.i < len(self.d) else 0) << self.nb
            self.i += 1
            self.nb += 8

    def bits(self, n):
        self.need(n)
        v = self.buf & ((1 << n) - 1)
        self.buf >>= n
        self.nb -= n
        return v

    def align(self):
        self.bits(self.nb & 7)

    def pos(self):
        """bits consumed from the start of the data"""
        return 8 * self.i - self.nb


def _table(lengths):
    """LSB-first lookup table over the next max-length bits -> (symbol, length)."""
    ml = max(lengths)
    counts = [0] * 16
    for n in lengths:
        counts[n] += 1
    counts[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + counts[b - 1]) << 1
        nxt[b] = code
    tab = [None] * (1 << ml)
    for s, n in enumerate(lengths):
        if n:
            c = nxt[n]
            nxt[n] += 1
            r = int(format(c, "0%db" % n)[::-1], 2)
            for hi in range(1 << (ml - n)):
                tab[r | (hi << n)] = (s, n)
    return tab, ml


def _decode(br, tab):
    t, ml = tab
    br.need(ml)
    s, n = t[br.buf & ((1 << ml) - 1)]
    br.buf >>= n
    br.nb -= n
    return s


_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
          12289, 16385, 24577]
_DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def trace(zstream):
    """zstream: a zlib stream.  Returns (blocks, data).  Each block is a dict: type ('stored' / 'fixed' / 'dynamic'),
    final, lit_lengths / dist_lengths / code_lengths (dynamic), symbols (ints for literals, (length, distance) for matches;
    the end of block is not listed), stored_len, and the bit positions in zstream of the block's first bit (start), of the
    first bit after its header (body: after the tree description of a dynamic block, after the 3 type bits of a fixed one)
    and of the first bit after the block (end)."""
    br = _Bits(zstream, 2)
    out = bytearray()
    blocks = []
    while True:
        start = br.pos()
        final, btype = br.bits(1), br.bits(2)
        blk = {"final": final, "symbols": [], "start": start}
        blocks.append(blk)
        if btype == 0:
            br.align()
            n, nn = br.bits(16), br.bits(16)
            assert n ^ nn == 0xffff
            blk.update(type="stored", stored_len=n)
            for _ in range(n):
                out.append(br.bits(8))
        else:
            if btype == 1:
                ll = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
                dl = [5] * 30
                blk["type"] = "fixed"
            else:
                hlit, hdist, hclen = br.bits(5) + 257, br.bits(5) + 1, br.bits(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[_ORDER[i]] = br.bits(3)
                ct = _table(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = _decode(br, ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.bits(2))
                    elif s == 17:
                        lens += [0] * (3 + br.bits(3))
                    else:
                        lens += [0] * (11 + br.bits(7))
                ll, dl = lens[:hlit], lens[hlit:]
                blk.update(type="dynamic", lit_lengths=ll, dist_lengths=dl, code_lengths=cl)
            blk["body"] = br.pos()
            lt, dt = _table(ll), _table(dl) if max(dl) else None
            while True:
                s = _decode(br, lt)
                if s < 256:
                    out.append(s)
                    blk["symbols"].append(s)
                elif s == 256:
                    break
                else:
                    c = s - 257
                    ln = _LBASE[c] + br.bits(_LEXT[c])
                    d = _decode(br, dt)
                    dist = _DBASE[d] + br.bits(_DEXT[d])
                    for _ in range(ln):
                        out.append(out[-dist])
                    blk["symbols"].append((ln, dist))
        blk["end"] = br.pos()
        if final:
            break
    br.align()
    assert zlib.adler32(bytes(out)) == int.from_bytes(zstream[br.i - br.nb // 8:br.i - br.nb // 8 + 4], "big")
    return blocks, bytes(out)


def first_difference(za, zb):
    """A readable description of where two zlib streams first differ, by block and symbol ("" when they decode alike)."""
    ba, _ = trace(za)
    bb, _ = trace(zb)
    for k, (x, y) in enumerate(zip(ba, bb)):
        for key in ("type", "final", "stored_len", "lit_lengths", "dist_lengths"):
            if x.get(key) != y.get(key):
                return "block %d: %s differs (%r vs %r)" % (k, key, x.get(key), y.get(key))
        for i, (s, t) in enumerate(zip(x["symbols"], y["symbols"])):
            if s != t:
                return "block %d symbol %d: %r vs %r" % (k, i, s, t)
        if len(x["symbols"]) != len(y["symbols"]):
            return "block %d: %d vs %d symbols" % (k, len(x["symbols"]), len(y["symbols"]))
    if len(ba) != len(bb):
        return "%d vs %d blocks" % (len(ba), len(bb))
    return ""
