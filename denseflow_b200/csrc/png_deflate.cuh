// png_deflate.cuh — the sequential pieces of zlib's deflate that the PNG encoder (png_encode.cu) restates per deflate block:
// the Huffman tree construction of trees.c (build_tree with its heap and depth tie-break, gen_bitlen with its overflow
// repair, gen_codes), the code-length tree (scan_tree / send_tree / build_bl_tree), the stored / fixed / dynamic choice of
// _tr_flush_block, and the symbol codes of compress_block.  Integer-only, callable from host and device, so one thread of a
// CTA builds a block's trees exactly as zlib's single thread does.
//
// The symbol stream is that of deflate_rle (strategy Z_RLE, which OpenCV's PNG encoder selects): literals and matches at
// distance 1 only.  A symbol is stored as a uint16: 0..255 a literal byte, 256 + (length - 3) a match, kSymEob the end of
// block.
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define PZ_HD __host__ __device__ __forceinline__
#else
#define PZ_HD inline
#endif

namespace dfb {
namespace pngz {

constexpr int kLCodes = 286;                    // literal / length codes (L_CODES)
constexpr int kDCodes = 30;                     // distance codes
constexpr int kBlCodes = 19;                    // code-length codes
constexpr int kHeapSize = 2 * kLCodes + 1;      // HEAP_SIZE
constexpr int kEndBlock = 256;
constexpr int kBlockSyms = 16383;               // lit_bufsize - 1 at memLevel 8: symbols per block before a flush
constexpr uint16_t kSymEob = 0xffff;
constexpr int kHdrWords = 144;                  // 3 + 14 + 19 * 3 + 316 * 14 bits of a dynamic header, rounded up

// zlib's ct_data: fc = frequency, later the (bit-reversed) code; dl = father node, later the code length
struct Ct {
    uint16_t fc, dl;
};

struct Trees {
    Ct ltree[kHeapSize];
    Ct dtree[2 * kDCodes + 1];
    Ct bltree[2 * kBlCodes + 1];
    int heap[kHeapSize];
    int heap_len, heap_max;
    uint8_t depth[kHeapSize];
    uint16_t bl_count[16];
    int64_t opt_len, static_len;
};

enum : uint32_t { kStored = 0, kFixed = 1, kDynamic = 2 };

// one deflate block as the emitter needs it
struct BlockInfo {
    uint32_t type;        // kStored / kFixed / kDynamic
    uint32_t hdr_bits;    // fixed / dynamic: block type bits + tree description, in hdr[]
    uint32_t bits;        // fixed / dynamic: every bit of the block (header, symbols, end of block)
    uint32_t pos, len;    // bytes of the uncompressed stream the block covers: [pos, pos + len)
    uint32_t first_sym, nsym;
    uint32_t last;        // BFINAL
    uint32_t dist;        // code of distance 1: bit-reversed code | length << 16
    uint32_t lit[kLCodes];  // literal / length codes: bit-reversed code | length << 16
    uint32_t hdr[kHdrWords];
};

// ---- the static tables of trees.c, in closed form ----
PZ_HD int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
PZ_HD int extra_lbits(int code) { return (code < 8 || code == 28) ? 0 : (code - 4) >> 2; }
// base_length[] of the length code; code 28 (length 258) has no extra bits and stands for lc = 255 alone
PZ_HD int base_length(int code) { return code < 8 ? code : code == 28 ? 255 : (4 + (code & 3)) << ((code - 4) >> 2); }
// _length_code[lc], lc = match length - 3 (0..255)
PZ_HD int length_code(int lc) {
    if (lc < 8) return lc;
    if (lc == 255) return 28;
    int lg = 3;
    while ((lc >> (lg + 1)) != 0) ++lg;
    const int k = lg - 2;
    return 4 * k + 4 + ((lc >> k) & 3);
}
PZ_HD int extra_dbits(int code) { return code < 4 ? 0 : (code - 2) >> 1; }
PZ_HD int extra_blbits(int n) { return n == 16 ? 2 : n == 17 ? 3 : n == 18 ? 7 : 0; }
PZ_HD int bl_order(int r) { return "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f"[r]; }

PZ_HD unsigned bi_reverse(unsigned code, int len) {
    unsigned res = 0;
    do {
        res |= code & 1;
        code >>= 1, res <<= 1;
    } while (--len > 0);
    return res >> 1;
}

// the canonical code gen_codes gives static_ltree, bit-reversed
PZ_HD uint32_t static_lcode(int n) {
    const unsigned c = n < 144 ? 0x30 + n : n < 256 ? 0x190 + (n - 144) : n < 280 ? n - 256 : 0xc0 + (n - 280);
    return bi_reverse(c, static_llen(n));
}

// ---- trees.c ----
// kind: 0 literal / length tree, 1 distance tree, 2 code-length tree
PZ_HD int tree_extra(int kind, int n) { return kind == 0 ? (n > 256 ? extra_lbits(n - 257) : 0) : kind == 1 ? extra_dbits(n) : extra_blbits(n); }
PZ_HD int tree_static_len(int kind, int n) { return kind == 0 ? static_llen(n) : 5; }

PZ_HD bool smaller(const Ct *t, int n, int m, const uint8_t *depth) {
    return t[n].fc < t[m].fc || (t[n].fc == t[m].fc && depth[n] <= depth[m]);
}

PZ_HD void pqdownheap(Trees &s, const Ct *tree, int k) {
    const int v = s.heap[k];
    int j = k << 1;
    while (j <= s.heap_len) {
        if (j < s.heap_len && smaller(tree, s.heap[j + 1], s.heap[j], s.depth)) j++;
        if (smaller(tree, v, s.heap[j], s.depth)) break;
        s.heap[k] = s.heap[j];
        k = j;
        j <<= 1;
    }
    s.heap[k] = v;
}

PZ_HD void gen_bitlen(Trees &s, Ct *tree, int max_code, int kind) {
    const int max_length = kind == 2 ? 7 : 15;
    int overflow = 0;
    for (int b = 0; b <= 15; b++) s.bl_count[b] = 0;
    tree[s.heap[s.heap_max]].dl = 0;  // root of the heap
    int h;
    for (h = s.heap_max + 1; h < kHeapSize; h++) {
        const int n = s.heap[h];
        int bits = tree[tree[n].dl].dl + 1;
        if (bits > max_length) bits = max_length, overflow++;
        tree[n].dl = (uint16_t)bits;
        if (n > max_code) continue;  // not a leaf
        s.bl_count[bits]++;
        const int xbits = tree_extra(kind, n);
        const int64_t f = tree[n].fc;
        s.opt_len += f * (bits + xbits);
        if (kind != 2) s.static_len += f * (tree_static_len(kind, n) + xbits);
    }
    if (overflow == 0) return;
    do {  // find the first bit length which could increase
        int bits = max_length - 1;
        while (s.bl_count[bits] == 0) bits--;
        s.bl_count[bits]--;
        s.bl_count[bits + 1] += 2;
        s.bl_count[max_length]--;
        overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; bits--) {  // recompute all lengths in increasing frequency
        int n = s.bl_count[bits];
        while (n != 0) {
            const int m = s.heap[--h];
            if (m > max_code) continue;
            if (tree[m].dl != (unsigned)bits) {
                s.opt_len += ((int64_t)bits - tree[m].dl) * tree[m].fc;
                tree[m].dl = (uint16_t)bits;
            }
            n--;
        }
    }
}

PZ_HD void gen_codes(Ct *tree, int max_code, const uint16_t *bl_count) {
    uint16_t next_code[16];
    unsigned code = 0;
    for (int bits = 1; bits <= 15; bits++) {
        code = (code + bl_count[bits - 1]) << 1;
        next_code[bits] = (uint16_t)code;
    }
    for (int n = 0; n <= max_code; n++) {
        const int len = tree[n].dl;
        if (len == 0) continue;
        tree[n].fc = (uint16_t)bi_reverse(next_code[len]++, len);
    }
}

// returns max_code
PZ_HD int build_tree(Trees &s, Ct *tree, int elems, int kind) {
    int max_code = -1;
    s.heap_len = 0, s.heap_max = kHeapSize;
    for (int n = 0; n < elems; n++) {
        if (tree[n].fc != 0) {
            s.heap[++s.heap_len] = max_code = n;
            s.depth[n] = 0;
        } else {
            tree[n].dl = 0;
        }
    }
    while (s.heap_len < 2) {  // at least two codes of non-zero frequency
        const int node = s.heap[++s.heap_len] = (max_code < 2 ? ++max_code : 0);
        tree[node].fc = 1;
        s.depth[node] = 0;
        s.opt_len--;
        if (kind != 2) s.static_len -= tree_static_len(kind, node);
    }
    for (int n = s.heap_len / 2; n >= 1; n--) pqdownheap(s, tree, n);
    int node = elems;
    do {
        const int n = s.heap[1];
        s.heap[1] = s.heap[s.heap_len--];
        pqdownheap(s, tree, 1);
        const int m = s.heap[1];
        s.heap[--s.heap_max] = n;
        s.heap[--s.heap_max] = m;
        tree[node].fc = (uint16_t)(tree[n].fc + tree[m].fc);
        s.depth[node] = (uint8_t)((s.depth[n] >= s.depth[m] ? s.depth[n] : s.depth[m]) + 1);
        tree[n].dl = tree[m].dl = (uint16_t)node;
        s.heap[1] = node++;
        pqdownheap(s, tree, 1);
    } while (s.heap_len >= 2);
    s.heap[--s.heap_max] = s.heap[1];
    gen_bitlen(s, tree, max_code, kind);
    gen_codes(tree, max_code, s.bl_count);
    return max_code;
}

PZ_HD void scan_tree(Trees &s, Ct *tree, int max_code) {
    int prevlen = -1, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) max_count = 138, min_count = 3;
    tree[max_code + 1].dl = 0xffff;  // guard
    for (int n = 0; n <= max_code; n++) {
        const int curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) {
            continue;
        } else if (count < min_count) {
            s.bltree[curlen].fc += count;
        } else if (curlen != 0) {
            if (curlen != prevlen) s.bltree[curlen].fc++;
            s.bltree[16].fc++;
        } else if (count <= 10) {
            s.bltree[17].fc++;
        } else {
            s.bltree[18].fc++;
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

// LSB-first bit writer into a word buffer the caller zeroed
struct BitWriter {
    uint32_t *w;
    uint32_t n = 0;
    PZ_HD void put(uint32_t v, int len) {
        if (len == 0) return;
        const uint32_t i = n >> 5, sh = n & 31;
        w[i] |= v << sh;
        if (sh + len > 32) w[i + 1] |= v >> (32 - sh);
        n += len;
    }
};

PZ_HD void send_tree(BitWriter &bw, const Trees &s, const Ct *tree, int max_code) {
    int prevlen = -1, nextlen = tree[0].dl, count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) max_count = 138, min_count = 3;
    auto code = [&](int c) { bw.put(s.bltree[c].fc, s.bltree[c].dl); };
    for (int n = 0; n <= max_code; n++) {
        const int curlen = nextlen;
        nextlen = tree[n + 1].dl;
        if (++count < max_count && curlen == nextlen) {
            continue;
        } else if (count < min_count) {
            do code(curlen);
            while (--count != 0);
        } else if (curlen != 0) {
            if (curlen != prevlen) {
                code(curlen);
                count--;
            }
            code(16);
            bw.put(count - 3, 2);
        } else if (count <= 10) {
            code(17);
            bw.put(count - 3, 3);
        } else {
            code(18);
            bw.put(count - 11, 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

// _tr_flush_block for one block whose literal / length frequencies (END_BLOCK's 1 included) are in s.ltree[].fc, distance
// frequencies in s.dtree[].fc, everything else of s zeroed.  stored_len: bytes the block covers.  Fills b (hdr[] zeroed by the
// caller) except pos / first_sym / nsym.
//
// zlib offers the stored block only while the block's bytes are still in its window (buf != NULL).  For the 32 KB window
// this fails only for blocks that cover more than 32 506 bytes (the window slides at strstart >= 2 * 32768 - 262), and such a
// block never qualifies: it has at most 16 383 symbols, a match costs at most 21 bits for at least 3 bytes and the
// dynamic code costs at most 9 bits per literal, so opt_len stays below 8 * stored_len.  The stored option is therefore
// taken whenever zlib's size test allows it.
PZ_HD void flush_block(Trees &s, uint32_t stored_len, bool last, BlockInfo &b) {
    const int lmax = build_tree(s, s.ltree, kLCodes, 0);
    const int dmax = build_tree(s, s.dtree, kDCodes, 1);
    scan_tree(s, s.ltree, lmax);
    scan_tree(s, s.dtree, dmax);
    build_tree(s, s.bltree, kBlCodes, 2);
    int max_blindex;
    for (max_blindex = kBlCodes - 1; max_blindex >= 3; max_blindex--)
        if (s.bltree[bl_order(max_blindex)].dl != 0) break;
    s.opt_len += 3 * ((int64_t)max_blindex + 1) + 5 + 5 + 4;
    int64_t opt_lenb = (s.opt_len + 3 + 7) >> 3;
    const int64_t static_lenb = (s.static_len + 3 + 7) >> 3;
    if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
    b.last = last;
    b.len = stored_len;
    if ((int64_t)stored_len + 4 <= opt_lenb) {
        b.type = kStored;
        b.hdr_bits = 0;
        b.bits = 0;
        return;
    }
    BitWriter bw{b.hdr};
    if (static_lenb == opt_lenb) {
        b.type = kFixed;
        bw.put((1u << 1) + last, 3);
        for (int n = 0; n < kLCodes; n++) b.lit[n] = static_lcode(n) | (uint32_t)static_llen(n) << 16;
        b.dist = 0u | 5u << 16;
        b.bits = (uint32_t)(3 + s.static_len);
    } else {
        b.type = kDynamic;
        bw.put((2u << 1) + last, 3);
        const int lcodes = lmax + 1, dcodes = dmax + 1, blcodes = max_blindex + 1;
        bw.put(lcodes - 257, 5);
        bw.put(dcodes - 1, 5);
        bw.put(blcodes - 4, 4);
        for (int r = 0; r < blcodes; r++) bw.put(s.bltree[bl_order(r)].dl, 3);
        send_tree(bw, s, s.ltree, lcodes - 1);
        send_tree(bw, s, s.dtree, dcodes - 1);
        for (int n = 0; n < kLCodes; n++) b.lit[n] = n <= lmax ? (s.ltree[n].fc | (uint32_t)s.ltree[n].dl << 16) : 0u;
        b.dist = s.dtree[0].fc | (uint32_t)s.dtree[0].dl << 16;
        b.bits = (uint32_t)(3 + s.opt_len);
    }
    b.hdr_bits = bw.n;
}

// the bits of one symbol under a block's codes (value LSB-first, returns the bit count)
PZ_HD int symbol_bits(uint16_t v, const uint32_t *lit, uint32_t dist, uint32_t &val) {
    if (v < 256 || v == kSymEob) {
        const uint32_t c = lit[v < 256 ? v : kEndBlock];
        val = c & 0xffff;
        return (int)(c >> 16);
    }
    const int lc = v - 256, code = length_code(lc), xb = extra_lbits(code);
    const uint32_t c = lit[257 + code];
    const int cl = (int)(c >> 16);
    val = (c & 0xffff) | ((uint32_t)(lc - base_length(code)) << cl) | ((dist & 0xffff) << (cl + xb));
    return cl + xb + (int)(dist >> 16);
}

// symbols of a maximal run of n equal bytes under deflate_rle: a literal, matches of min(left, 258) while at least 3 bytes
// are left, then 0..2 literals
PZ_HD uint32_t run_matches(uint32_t n) { return n >= 4 ? (n - 4) / 258 + 1 : 0; }
PZ_HD uint32_t run_symbols(uint32_t n) {
    const uint32_t r = n - 1, m = run_matches(n);
    const uint32_t k = m ? (r < 258 * m ? r : 258 * m) : 0;
    return 1 + m + (r - k);
}

// ---- zlib container / PNG helpers ----
constexpr uint32_t kAdlerMod = 65521;
constexpr uint32_t kCrcPoly = 0xedb88320u;

// a * b modulo the CRC-32 polynomial, reflected (zlib's multmodp)
PZ_HD uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ kCrcPoly : b >> 1;
    }
    return p;
}
// x^(8 n) modulo the polynomial: the operator that runs a CRC register over n zero bytes
PZ_HD uint32_t x8nmodp(uint64_t n) {
    uint32_t p = 1u << 31, sq = 1u << 23;  // x^0, x^8
    while (n) {
        if (n & 1) p = multmodp(sq, p);
        sq = multmodp(sq, sq);
        n >>= 1;
    }
    return p;
}

}  // namespace pngz
}  // namespace dfb
