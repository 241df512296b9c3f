// A host build of the deflate block code the GPU PNG encoder runs per block (denseflow_b200/csrc/png_deflate.cuh, which is
// host-callable): tests/test_png_deflate_cpu.py compiles it with the system C++ compiler and compares flush_block with
// zlib on every block of every case in tests/deflate_cases.py.
#include <string.h>

#include "png_deflate.cuh"

using namespace dfb::pngz;

// lfreq: 286 literal / length frequencies (END_BLOCK's 1 included), dfreq: 30 distance frequencies.  out: type, hdr_bits,
// bits, the length of distance code 0, the literal tree's max_code; sizes: opt_len, static_len as flush_block leaves them;
// lit_len: 286 code lengths of the block as sent; tree_len: 286 lengths of the literal / length tree built (also when the
// block is sent stored or fixed); hdr: kHdrWords words of header bits.
extern "C" int pngz_flush_block(const uint32_t *lfreq, const uint32_t *dfreq, uint32_t stored_len, int last, uint32_t *out,
                                int64_t *sizes, uint32_t *lit_len, uint32_t *tree_len, uint32_t *hdr) {
    static Trees s;
    static BlockInfo b;
    memset(&s, 0, sizeof s);
    memset(&b, 0, sizeof b);
    for (int n = 0; n < kLCodes; n++) s.ltree[n].fc = (uint16_t)lfreq[n];
    for (int n = 0; n < kDCodes; n++) s.dtree[n].fc = (uint16_t)dfreq[n];
    flush_block(s, stored_len, last != 0, b);
    out[0] = b.type;
    out[1] = b.hdr_bits;
    out[2] = b.bits;
    out[3] = b.dist >> 16;
    int lmax = 0;
    while (s.ltree[lmax + 1].dl != 0xffff) lmax++;  // scan_tree's guard follows max_code
    out[4] = (uint32_t)lmax;
    sizes[0] = s.opt_len;
    sizes[1] = s.static_len;
    for (int n = 0; n < kLCodes; n++) lit_len[n] = b.lit[n] >> 16;
    for (int n = 0; n < kLCodes; n++) tree_len[n] = n <= lmax ? s.ltree[n].dl : 0;
    memcpy(hdr, b.hdr, sizeof b.hdr);
    return kHdrWords;
}
