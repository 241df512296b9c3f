"""zlib's block sizing restated from a block's symbol histogram: build_tree (heap, depth tie-break, the fake nodes of a tree
with fewer than two symbols), gen_bitlen with its overflow repair, scan_tree, the max_blindex floor of 4 and
_tr_flush_block's stored / fixed / dynamic choice (trees.c).  Pinned to zlib's own streams in tests/test_png_deflate_cpu.py;
the tests use it to find the block-choice ties and to assert which edge a case reaches.  Blocks come from the Z_RLE parse
of a scanline stream, 16 383 symbols each, as deflate_rle flushes them."""
import numpy as np

L_CODES, D_CODES, BL_CODES = 286, 30, 19
HEAP_SIZE = 2 * L_CODES + 1
BLOCK_SYMS = 16383
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
EXTRA_LBITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
EXTRA_DBITS = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
KINDS = {"lit": (L_CODES, 15, 257, EXTRA_LBITS), "dist": (D_CODES, 15, 0, EXTRA_DBITS), "bl": (BL_CODES, 7, 0, EXTRA_BLBITS)}


def static_len(kind, n):
    if kind == "dist":
        return 5
    return 8 if n < 144 else 9 if n < 256 else 7 if n < 280 else 8


def length_code(length):
    """the literal / length symbol (257..285) of a match length (3..258)"""
    lc = length - 3
    if lc == 255:
        return 285
    if lc < 8:
        return 257 + lc
    k = lc.bit_length() - 3
    return 257 + 4 * k + 4 + ((lc >> k) & 3)


def build_tree(freq, kind, st):
    """One tree from its symbol frequencies.  st: the block's running {"opt_len", "static_len"}, updated as zlib does.
    Returns lengths (per symbol), max_code, fake (the fake nodes added), depth (the deepest leaf before the repair) and
    overflow (leaves the repair had to move)."""
    elems, max_length, base, extra = KINDS[kind]
    fc = list(freq) + [0] * (2 * elems + 1 - len(freq))
    dad, depth, raw = [0] * len(fc), [0] * len(fc), [0] * len(fc)
    heap = [0] * (HEAP_SIZE + 1)
    heap_len, heap_max, max_code, fake = 0, HEAP_SIZE, -1, []
    for n in range(elems):
        if fc[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
    while heap_len < 2:
        node = max_code + 1 if max_code < 2 else 0
        max_code = max(max_code, node)
        heap_len += 1
        heap[heap_len] = node
        fc[node] = 1
        fake.append(node)
        st["opt_len"] -= 1
        if kind != "bl":
            st["static_len"] -= static_len(kind, node)

    def smaller(n, m):
        return fc[n] < fc[m] or (fc[n] == fc[m] and depth[n] <= depth[m])

    def down(k):
        v, j = heap[k], 2 * k
        while j <= heap_len:
            if j < heap_len and smaller(heap[j + 1], heap[j]):
                j += 1
            if smaller(v, heap[j]):
                break
            heap[k], k, j = heap[j], j, 2 * j
        heap[k] = v

    for k in range(heap_len // 2, 0, -1):
        down(k)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[heap_len]
        heap_len -= 1
        down(1)
        m = heap[1]
        heap_max -= 2
        heap[heap_max + 1], heap[heap_max] = n, m
        fc[node] = fc[n] + fc[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        down(1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]
    # gen_bitlen
    ln = [0] * len(fc)
    bl_count, overflow = [0] * 16, 0
    for h in range(heap_max + 1, HEAP_SIZE):
        n = heap[h]
        raw[n] = raw[dad[n]] + 1
        bits = ln[dad[n]] + 1
        if bits > max_length:
            bits, overflow = max_length, overflow + 1
        ln[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xbits = extra[n - base] if n >= base else 0
        st["opt_len"] += fc[n] * (bits + xbits)
        if kind != "bl":
            st["static_len"] += fc[n] * (static_len(kind, n) + xbits)
    moved = overflow
    if overflow:
        while overflow > 0:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
        h = HEAP_SIZE
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if ln[m] != bits:
                    st["opt_len"] += (bits - ln[m]) * fc[m]
                    ln[m] = bits
                n -= 1
    leaves = range(max_code + 1)
    return {"lengths": [ln[n] if fc[n] else 0 for n in leaves] + [0] * (elems - max_code - 1), "max_code": max_code,
            "fake": fake, "depth": max(raw[n] for n in leaves if fc[n]), "overflow": moved}


def scan_tree(lengths, max_code, blfreq):
    prevlen, nextlen, count = -1, lengths[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        curlen, nextlen = nextlen, lengths[n + 1] if n + 1 <= max_code else 0xffff
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            blfreq[curlen] += count
        elif curlen != 0:
            if curlen != prevlen:
                blfreq[curlen] += 1
            blfreq[16] += 1
        elif count <= 10:
            blfreq[17] += 1
        else:
            blfreq[18] += 1
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4


def flush_block(lfreq, dfreq, stored_len):
    """_tr_flush_block at level 1.  lfreq: 286 literal / length frequencies (END_BLOCK's 1 included), dfreq: 30 distance
    frequencies, stored_len: bytes the block covers.  Returns the three trees, the sizes and the chosen type."""
    st = {"opt_len": 0, "static_len": 0}
    lt = build_tree(lfreq, "lit", st)
    dt = build_tree(dfreq, "dist", st)
    blfreq = [0] * BL_CODES
    scan_tree(lt["lengths"], lt["max_code"], blfreq)
    scan_tree(dt["lengths"], dt["max_code"], blfreq)
    bt = build_tree(blfreq, "bl", st)
    max_blindex = next(i for i in range(BL_CODES - 1, 2, -1) if bt["lengths"][BL_ORDER[i]] or i == 3)
    opt_len = st["opt_len"] + 3 * (max_blindex + 1) + 5 + 5 + 4
    opt_lenb = dyn_lenb = (opt_len + 3 + 7) >> 3
    static_lenb = (st["static_len"] + 3 + 7) >> 3
    if static_lenb <= opt_lenb:
        opt_lenb = static_lenb
    kind = "stored" if stored_len + 4 <= opt_lenb else "fixed" if static_lenb == opt_lenb else "dynamic"
    return {"type": kind, "lit": lt, "dist": dt, "bl": bt, "max_blindex": max_blindex, "opt_len": opt_len,
            "static_len": st["static_len"], "dyn_lenb": dyn_lenb, "static_lenb": static_lenb, "stored_len": stored_len,
            "bits": 3 + (opt_len if kind == "dynamic" else st["static_len"])}


def symbols(raw):
    """deflate_rle's parse of raw (tests/png_cases.rle_parse, vectorised): per symbol its literal / length code and the
    bytes it covers"""
    a = np.frombuffer(bytes(raw), np.uint8)
    starts = np.flatnonzero(np.r_[True, a[1:] != a[:-1]])
    n = np.diff(np.r_[starts, len(a)])
    r = n - 1
    m = np.where(n >= 4, (n - 4) // 258 + 1, 0)
    k = np.minimum(r, 258 * m)
    cnt = 1 + m + (r - k)
    rid = np.repeat(np.arange(len(n)), cnt)
    j = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    mm = m[rid]
    is_match = (j >= 1) & (j <= mm)
    mlen = np.where(j < mm, 258, k[rid] - 258 * (mm - 1))
    lens = np.where(is_match, mlen, 1)
    table = np.array([0, 0, 0] + [length_code(x) for x in range(3, 259)])
    code = np.where(is_match, table[np.where(is_match, mlen, 0)], a[starts][rid])
    return code, lens


def block_histograms(raw):
    """(lfreq, dfreq, stored_len, nsym) of every deflate block of the stream, the empty final block included"""
    code, lens = symbols(raw)
    nb = len(code) // BLOCK_SYMS + 1
    b = np.arange(len(code)) // BLOCK_SYMS
    lf = np.bincount(b * L_CODES + code, minlength=nb * L_CODES).reshape(nb, L_CODES)
    lf[:, 256] = 1
    dist = np.bincount(b, weights=code > 256, minlength=nb).astype(int)
    stored = np.bincount(b, weights=lens, minlength=nb).astype(int)
    nsym = np.bincount(b, minlength=nb)
    return [(lf[i].tolist(), [int(dist[i])] + [0] * (D_CODES - 1), int(stored[i]), int(nsym[i])) for i in range(nb)]


def blocks(raw):
    """flush_block of every block of raw's zlib stream, with its histogram"""
    out = []
    for lf, df, stored, nsym in block_histograms(raw):
        blk = flush_block(lf, df, stored)
        blk.update(lfreq=lf, dfreq=df, nsym=nsym)
        out.append(blk)
    return out
