// jpeg_encode.cu — imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q]) on the GPU, byte for byte: the JPEG files of
// encodeFlowMap (src/common.cpp:48-64 of the reference, one gray component) and of the frame extraction
// (src/denseflow_gpu.cpp:82-105, YCbCr 4:2:0).  OpenCV's defaults make libjpeg-turbo's compressor run one configuration:
// baseline, the standard (Annex K) Huffman tables, jpeg_fdct_islow, quality-scaled Annex K quantisers, no restart markers.
// All of it is integer arithmetic, restated here exactly; tests/jpeg_encode_restate.py is its numpy counterpart.
//
// A batch of n images of one size is encoded by one sequence of launches, blockIdx.y spanning the images:
//   k_dct      one thread per 8 x 8 block in MCU order: edge-replicated samples, islow DCT, libjpeg-turbo's quantize
//              (reciprocal, correction, shift over quantval << 3), the coefficients in zig-zag order, their nonzero mask,
//              the quantised DC and the AC bit count.  4:2:0 luma blocks past the component's blocks are dummy blocks
//   k_dc       one thread per block: DC difference (dummy blocks copy their DC as compress_data does), bit count; the
//              bit count of each CTA's tile of blocks
//   k_bits     one CTA per image: exclusive scan of the tile bit counts, capacity check
//   k_offsets  one CTA per tile: bit offset of every block; zeroes the words blocks share
//   k_emit     one thread per block: its codes at its bit offset (MSB first); words inside its range stored, edge words
//              ORed; the last block pads the final byte with 1-bits (flush_bits)
//   k_ff_count per 1 KB tile of entropy data: 0xFF bytes
//   k_ff_scan  one CTA per image: tile bases of the stuffed zeros, file length, capacity check
//   k_scatter  per tile: header (tile 0), data with a 0x00 after every 0xFF, EOI (last tile)
#include <algorithm>
#include <stdexcept>
#include <string>

#include "block_scan.cuh"
#include "common.cuh"
#include "jpeg_encode.h"

namespace dfb {

namespace {

constexpr size_t kWorkspaceBudget = size_t(512) << 20;  // images per launch sequence are capped by this much workspace
constexpr int kBlkThreads = 128;
constexpr int kTileThreads = 256;
constexpr int kTileBytes = 4 * kTileThreads;  // one word per thread

// ---- Annex K tables ----
constexpr uint8_t kStdLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                   14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                   18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                   49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kStdChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                     99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
#define DFB_ZIGZAG                                                                                                          \
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, \
        42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,  \
        62, 63
constexpr uint8_t kZigzag[64] = {DFB_ZIGZAG};  // zig-zag index -> natural index

struct HuffSpec {
    uint8_t bits[16];
    uint8_t vals[162];
    int nvals;
};
constexpr HuffSpec kDcLuma = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
constexpr HuffSpec kDcChroma = {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
constexpr HuffSpec kAcLuma = {
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    162};
constexpr HuffSpec kAcChroma = {
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    162};

// jpeg_make_c_derived_tbl: symbol -> code << 8 | length (0: no code), [0] luminance, [1] chrominance
struct HuffTabs {
    uint32_t dc[2][16];
    uint32_t ac[2][256];
};
constexpr void derive(const HuffSpec &s, uint32_t *out) {
    uint32_t code = 0;
    int k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < s.bits[l - 1]; ++i) out[s.vals[k++]] = code++ << 8 | (uint32_t)l;
        code <<= 1;
    }
}
constexpr HuffTabs make_huff() {
    HuffTabs t{};
    derive(kDcLuma, t.dc[0]);
    derive(kDcChroma, t.dc[1]);
    derive(kAcLuma, t.ac[0]);
    derive(kAcChroma, t.ac[1]);
    return t;
}
__device__ const HuffTabs g_huff = make_huff();

// compute_reciprocal (jcdctmgr.c, 16-bit DCTELEM) of every quantiser step, natural order: rc = reciprocal | correction << 16
struct QuantTabs {
    uint32_t rc[2][64];
    uint8_t sh[2][64];
};

int quality_scale(int q) {  // jpeg_quality_scaling
    q = std::min(std::max(q, 1), 100);
    return q < 50 ? 5000 / q : 200 - 2 * q;
}
int quant_step(int basic, int quality) {  // jpeg_add_quant_table, force_baseline
    return std::min(std::max((basic * quality_scale(quality) + 50) / 100, 1), 255);
}

QuantTabs make_quant(int quality) {
    QuantTabs t{};
    for (int c = 0; c < 2; ++c)
        for (int i = 0; i < 64; ++i) {
            const uint32_t d = (uint32_t)quant_step((c ? kStdChromaQ : kStdLumaQ)[i], quality) << 3;
            int b = 31 - __builtin_clz(d), r = 16 + b;
            uint32_t fq = (uint32_t)((1ull << r) / d), fr = (uint32_t)((1ull << r) % d), corr = d / 2;
            if (fr == 0) {
                fq >>= 1;
                --r;
            } else if (fr <= d / 2) {
                ++corr;
            } else {
                ++fq;
            }
            t.rc[c][i] = fq | corr << 16;
            t.sh[c][i] = (uint8_t)r;
        }
    return t;
}

// every byte before the entropy-coded data: SOI, JFIF APP0 1.01, DQT per table, SOF0, DHT (DC, AC per table), SOS
struct Header {
    uint32_t len;
    uint8_t b[628];
};

Header make_header(int w, int h, int comps, int quality) {
    Header hd{};
    uint32_t n = 0;
    auto put = [&](std::initializer_list<int> v) {
        for (int x : v) hd.b[n++] = (uint8_t)x;
    };
    put({0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
    for (int c = 0; c < (comps == 3 ? 2 : 1); ++c) {
        put({0xFF, 0xDB, 0, 67, c});
        for (int k = 0; k < 64; ++k) hd.b[n++] = (uint8_t)quant_step((c ? kStdChromaQ : kStdLumaQ)[kZigzag[k]], quality);
    }
    put({0xFF, 0xC0, 0, 8 + 3 * comps, 8, h >> 8, h & 255, w >> 8, w & 255, comps});
    if (comps == 1) put({1, 0x11, 0});
    else put({1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
    for (int c = 0; c < (comps == 3 ? 2 : 1); ++c)
        for (int ac = 0; ac < 2; ++ac) {
            const HuffSpec &s = ac ? (c ? kAcChroma : kAcLuma) : (c ? kDcChroma : kDcLuma);
            const int len = 2 + 1 + 16 + s.nvals;
            put({0xFF, 0xC4, len >> 8, len & 255, ac << 4 | c});
            for (int i = 0; i < 16; ++i) hd.b[n++] = s.bits[i];
            for (int i = 0; i < s.nvals; ++i) hd.b[n++] = s.vals[i];
        }
    put({0xFF, 0xDA, 0, 6 + 2 * comps, comps});
    if (comps == 1) put({1, 0x00});
    else put({1, 0x00, 2, 0x11, 3, 0x11});
    put({0, 63, 0});
    hd.len = n;
    return hd;
}

struct ImgInfo {
    uint64_t bits;  // entropy bits including the final 1-bit padding
    uint32_t pad, error, tiles, ff;
};

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Geometry and per-image workspace layout of a batch (all images have the same size)
struct Geo {
    int w, h, comps, wb, hb, mx, my, ccols, crows;
    uint32_t nblk, btiles, tiles_max;
    uint64_t cap, ewords;
    size_t o_coef, o_mask, o_dc, o_acb, o_bits, o_tile, o_diff, o_off, o_ent, o_tcnt, o_info, bytes;

    Geo(int comps_, int w_, int h_, size_t cap_) {
        comps = comps_, w = w_, h = h_, cap = cap_;
        wb = ceil_div(w, 8), hb = ceil_div(h, 8), mx = ceil_div(w, 16), my = ceil_div(h, 16);
        ccols = jpeg_chroma_cols(w), crows = (h + 1) / 2;
        nblk = comps == 1 ? (uint32_t)wb * hb : (uint32_t)mx * my * 6;
        btiles = (nblk + kBlkThreads - 1) / kBlkThreads;
        ewords = cap / 4 + 2;
        tiles_max = (uint32_t)((cap + kTileBytes - 1) / kTileBytes);
        size_t o = 0;
        o_coef = o, o = align256(o + 128 * (size_t)nblk);
        o_mask = o, o = align256(o + 8 * (size_t)nblk);
        o_dc = o, o = align256(o + 4 * (size_t)nblk);
        o_acb = o, o = align256(o + 4 * (size_t)nblk);
        o_bits = o, o = align256(o + 4 * (size_t)nblk);
        o_tile = o, o = align256(o + 8 * (size_t)btiles);
        o_diff = o, o = align256(o + 4 * (size_t)nblk);
        o_off = o, o = align256(o + 8 * (size_t)nblk);
        o_ent = o, o = align256(o + 4 * ewords);
        o_tcnt = o, o = align256(o + 4 * (size_t)tiles_max + 4);
        o_info = o, o = align256(o + sizeof(ImgInfo));
        bytes = o;
    }
    template <typename T> __device__ T *at(uint8_t *ws, int img, size_t off) const { return reinterpret_cast<T *>(ws + (size_t)img * bytes + off); }

    // block b of the encode order: component, its block coordinates, and whether it is a dummy block
    __device__ void block(uint32_t b, int &comp, int &k, uint32_t &m, int &bx, int &by, bool &dummy) const {
        if (comps == 1) {
            comp = 0, k = 0, m = b, bx = (int)(b % (uint32_t)wb), by = (int)(b / (uint32_t)wb), dummy = false;
            return;
        }
        m = b / 6, k = (int)(b - 6 * m);
        const int mxx = (int)(m % (uint32_t)mx), myy = (int)(m / (uint32_t)mx);
        if (k < 4) {
            comp = 0, bx = 2 * mxx + (k & 1), by = 2 * myy + (k >> 1);
            dummy = bx >= wb || by >= hb;
        } else {
            comp = k - 3, bx = mxx, by = myy, dummy = false;
        }
    }
};

__device__ __forceinline__ int category(int v) { return 32 - __clz(abs(v)); }

// jpeg_fdct_islow (jfdctint.c) on 8 elements S apart.  Pass 1 (rows) leaves the outputs scaled up by PASS1_BITS = 2.
template <int S, bool P1> __device__ __forceinline__ void fdct8(int *d) {
    const int tmp0 = d[0] + d[7 * S], tmp7 = d[0] - d[7 * S];
    const int tmp1 = d[S] + d[6 * S], tmp6 = d[S] - d[6 * S];
    const int tmp2 = d[2 * S] + d[5 * S], tmp5 = d[2 * S] - d[5 * S];
    const int tmp3 = d[3 * S] + d[4 * S], tmp4 = d[3 * S] - d[4 * S];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    constexpr int n = P1 ? 13 - 2 : 13 + 2, R = 1 << (n - 1);
    if (P1) {
        d[0] = (tmp10 + tmp11) * 4;
        d[4 * S] = (tmp10 - tmp11) * 4;
    } else {
        d[0] = (tmp10 + tmp11 + 2) >> 2;
        d[4 * S] = (tmp10 - tmp11 + 2) >> 2;
    }
    int z1 = (tmp12 + tmp13) * 4433;
    d[2 * S] = (z1 + tmp13 * 6270 + R) >> n;
    d[6 * S] = (z1 - tmp12 * 15137 + R) >> n;
    z1 = tmp4 + tmp7;
    int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int z5 = (z3 + z4) * 9633;
    z1 *= -7373;
    z2 *= -20995;
    z3 = z3 * -16069 + z5;
    z4 = z4 * -3196 + z5;
    d[7 * S] = (tmp4 * 2446 + z1 + z3 + R) >> n;
    d[5 * S] = (tmp5 * 16819 + z2 + z4 + R) >> n;
    d[3 * S] = (tmp6 * 25172 + z2 + z3 + R) >> n;
    d[S] = (tmp7 * 12299 + z1 + z4 + R) >> n;
}

__global__ void __launch_bounds__(kBlkThreads) k_dct(JpegSrc src, uint8_t *ws, Geo G, QuantTabs Q) {
    const int img = blockIdx.y;
    __shared__ uint8_t acsz[2][256];
    for (int i = threadIdx.x; i < 512; i += kBlkThreads) acsz[i >> 8][i & 255] = (uint8_t)g_huff.ac[i >> 8][i & 255];
    __syncthreads();
    const uint32_t b = blockIdx.x * kBlkThreads + threadIdx.x;
    if (b >= G.nblk) return;
    int comp, k, bx, by;
    uint32_t m;
    bool dummy;
    G.block(b, comp, k, m, bx, by, dummy);
    const int t = comp > 0;
    uint4 *coef = G.at<uint4>(ws, img, G.o_coef) + (size_t)b * 8;
    if (dummy) {  // AC zero; its DC is set by k_dc
#pragma unroll
        for (int i = 0; i < 8; ++i) coef[i] = make_uint4(0, 0, 0, 0);
        G.at<uint64_t>(ws, img, G.o_mask)[b] = 0;
        G.at<int>(ws, img, G.o_dc)[b] = 0;
        G.at<uint32_t>(ws, img, G.o_acb)[b] = acsz[0][0];
        return;
    }
    const uint8_t *p = src.base + (size_t)img * src.img_stride;
    size_t pitch = src.pitch;
    int pw = G.w, ph = G.h;
    if (comp) {
        p += comp == 1 ? src.cb_off : src.cr_off;
        pitch = src.c_pitch, pw = G.ccols, ph = G.crows;
    }
    int d[64];
    int cols[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) cols[c] = min(8 * bx + c, pw - 1);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const uint8_t *row = p + (size_t)min(8 * by + r, ph - 1) * pitch;
#pragma unroll
        for (int c = 0; c < 8; ++c) d[8 * r + c] = (int)row[cols[c]] - 128;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) fdct8<1, true>(d + 8 * r);
#pragma unroll
    for (int c = 0; c < 8; ++c) fdct8<8, false>(d + c);
    // quantize (jcdctmgr.c) as written, then zig-zag order
    constexpr int nat[64] = {DFB_ZIGZAG};
    int zz[64];
#pragma unroll
    for (int z = 0; z < 64; ++z) {
        const int i = nat[z], v = d[i];
        const uint32_t rc = Q.rc[t][i];
        const int q = (int)((((uint32_t)abs(v) + (rc >> 16)) * (rc & 0xffff)) >> Q.sh[t][i]);
        zz[z] = v < 0 ? -q : q;
    }
    uint64_t mask = 0;
    uint32_t bits = 0;
    int run = 0;
#pragma unroll
    for (int z = 1; z < 64; ++z) {
        if (zz[z] == 0) {
            ++run;
        } else {
            mask |= 1ull << z;
            for (; run > 15; run -= 16) bits += acsz[t][0xF0];
            const int n = category(zz[z]);
            bits += acsz[t][run << 4 | n] + n;
            run = 0;
        }
    }
    if (run) bits += acsz[t][0];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = (uint32_t)(zz[8 * i + 2 * j] & 0xffff) | (uint32_t)zz[8 * i + 2 * j + 1] << 16;
        coef[i] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    G.at<uint64_t>(ws, img, G.o_mask)[b] = mask;
    G.at<int>(ws, img, G.o_dc)[b] = zz[0];
    G.at<uint32_t>(ws, img, G.o_acb)[b] = bits;
}

// quantised DC of block b; a dummy luma block copies it as compress_data (jccoefct.c) does: from the block to its left,
// and in the bottom MCU row from the last block of the row above (Y01, itself a copy of Y00 past the right edge)
__device__ __forceinline__ int dc_of(const Geo &G, const int *dc, uint32_t b) {
    if (G.comps == 1) return dc[b];
    int comp, k, bx, by;
    uint32_t m;
    bool dummy;
    G.block(b, comp, k, m, bx, by, dummy);
    if (!dummy) return dc[b];
    const uint32_t b0 = 6 * m;
    const int y01 = 2 * (int)(m % (uint32_t)G.mx) + 1 >= G.wb ? dc[b0] : dc[b0 + 1];
    if (k == 1) return dc[b0];
    if (k == 2 || by >= G.hb) return y01;
    return dc[b0 + 2];
}

// the previous block of b's component in encode order, or -1
__device__ __forceinline__ int64_t prev_of(const Geo &G, uint32_t b) {
    if (G.comps == 1) return (int64_t)b - 1;
    const uint32_t k = b % 6;
    if (k >= 4) return b >= 6 ? (int64_t)b - 6 : -1;
    if (k > 0) return (int64_t)b - 1;
    return b >= 6 ? (int64_t)b - 3 : -1;
}

// one thread per block: its DC difference and its bit count (DC code + AC bits)
__global__ void __launch_bounds__(kBlkThreads) k_dc(uint8_t *ws, Geo G) {
    const int img = blockIdx.y;
    __shared__ uint8_t dcsz[2][16];
    if (threadIdx.x < 32) dcsz[threadIdx.x >> 4][threadIdx.x & 15] = (uint8_t)g_huff.dc[threadIdx.x >> 4][threadIdx.x & 15];
    __syncthreads();
    const uint32_t b = blockIdx.x * kBlkThreads + threadIdx.x;
    uint32_t bits = 0;
    if (b < G.nblk) {
        const int *dc = G.at<int>(ws, img, G.o_dc);
        const int64_t p = prev_of(G, b);
        const int diff = dc_of(G, dc, b) - (p >= 0 ? dc_of(G, dc, (uint32_t)p) : 0);
        const int n = category(diff);
        const int t = G.comps == 3 && b % 6 >= 4;
        bits = dcsz[t][n] + n + G.at<uint32_t>(ws, img, G.o_acb)[b];
        G.at<int>(ws, img, G.o_diff)[b] = diff;
        G.at<uint32_t>(ws, img, G.o_bits)[b] = bits;
    }
    __shared__ uint32_t sm[kBlkThreads / 32];
    const uint32_t tile = block_sum<kBlkThreads>(bits, sm);
    if (threadIdx.x == 0) G.at<uint64_t>(ws, img, G.o_tile)[blockIdx.x] = tile;
}

// one CTA per image: exclusive scan of the tile bit counts (k_dc's CTAs) into tile bit offsets, the capacity check
__global__ void __launch_bounds__(1024) k_bits(uint8_t *ws, Geo G, uint32_t hdr_len, uint64_t *lens) {
    const int img = blockIdx.x;
    __shared__ uint64_t sm[32];
    uint64_t *tiles = G.at<uint64_t>(ws, img, G.o_tile);
    const uint32_t T = G.btiles, per = (T + 1023) / 1024, lo = min(T, threadIdx.x * per), hi = min(T, lo + per);
    uint64_t sum = 0;
    for (uint32_t i = lo; i < hi; ++i) sum += tiles[i];
    uint64_t total;
    uint64_t o = block_scan<1024>(sum, total, sm);
    const uint32_t pad = (uint32_t)(-total & 7);
    const uint64_t E = (total + pad) / 8, need = hdr_len + E + 2;
    ImgInfo *info = G.at<ImgInfo>(ws, img, G.o_info);
    if (need > G.cap) {  // the file cannot fit: report the length without the stuffed zeros, write nothing
        if (threadIdx.x == 0) {
            info->error = 1;
            lens[img] = need | kJpegLenLowerBound;
        }
        return;
    }
    for (uint32_t i = lo; i < hi; ++i) {
        const uint64_t v = tiles[i];
        tiles[i] = o;
        o += v;
    }
    if (threadIdx.x == 0) {
        G.at<uint32_t>(ws, img, G.o_ent)[(total + pad) >> 5] = 0;  // the last block's final partial word
        info->bits = total + pad;
        info->pad = pad;
        info->error = 0;
        info->tiles = (uint32_t)((E + kTileBytes - 1) / kTileBytes);
    }
}

// one CTA per tile of k_dc: bit offset of every block; zeroes the word each block starts in (shared with the block before,
// k_emit ORs into it)
__global__ void __launch_bounds__(kBlkThreads) k_offsets(uint8_t *ws, Geo G) {
    const int img = blockIdx.y;
    if (G.at<ImgInfo>(ws, img, G.o_info)->error) return;
    const uint32_t b = blockIdx.x * kBlkThreads + threadIdx.x;
    const uint32_t bits = b < G.nblk ? G.at<uint32_t>(ws, img, G.o_bits)[b] : 0;
    __shared__ uint32_t sm[kBlkThreads / 32];
    uint32_t total;
    const uint64_t o = G.at<uint64_t>(ws, img, G.o_tile)[blockIdx.x] + block_scan<kBlkThreads>(bits, total, sm);
    if (b >= G.nblk) return;
    G.at<uint64_t>(ws, img, G.o_off)[b] = o;
    G.at<uint32_t>(ws, img, G.o_ent)[o >> 5] = 0;
}

// MSB-first bit writer over 32-bit words (bit 31 first); the first word is shared with the block before unless the block
// starts on a word, the last one with the block after
struct BitWriter {
    uint32_t *w;
    uint64_t wi, lim, acc;
    int n;
    bool shared;
    __device__ BitWriter(uint32_t *words, uint64_t off, uint64_t limit) : w(words), wi(off >> 5), lim(limit), acc(0), n((int)(off & 31)), shared((off & 31) != 0) {}
    __device__ __forceinline__ void put(uint32_t v, int len) {
        acc = acc << len | v;
        n += len;
        if (n >= 32) {
            n -= 32;
            const uint32_t word = (uint32_t)(acc >> n);
            if (wi < lim) {
                if (shared) atomicOr(&w[wi], word);
                else w[wi] = word;
            }
            shared = false;
            ++wi;
            acc &= (1ull << n) - 1;
        }
    }
    __device__ __forceinline__ void code(uint32_t e) { put(e >> 8, (int)(e & 0xff)); }
    __device__ __forceinline__ void finish() {
        if (n && wi < lim) atomicOr(&w[wi], (uint32_t)(acc << (32 - n)));
    }
};

__global__ void __launch_bounds__(kBlkThreads) k_emit(uint8_t *ws, Geo G) {
    const int img = blockIdx.y;
    const ImgInfo *info = G.at<ImgInfo>(ws, img, G.o_info);
    if (info->error) return;
    __shared__ HuffTabs tabs;
    for (int i = threadIdx.x; i < (int)(sizeof(HuffTabs) / 4); i += kBlkThreads)
        reinterpret_cast<uint32_t *>(&tabs)[i] = reinterpret_cast<const uint32_t *>(&g_huff)[i];
    __syncthreads();
    const uint32_t b = blockIdx.x * kBlkThreads + threadIdx.x;
    if (b >= G.nblk) return;
    const int t = G.comps == 3 && b % 6 >= 4;
    BitWriter W(G.at<uint32_t>(ws, img, G.o_ent), G.at<uint64_t>(ws, img, G.o_off)[b], G.ewords);
    const int diff = G.at<int>(ws, img, G.o_diff)[b];
    int n = category(diff);
    W.code(tabs.dc[t][n]);
    if (n) W.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
    uint64_t mask = G.at<uint64_t>(ws, img, G.o_mask)[b];
    const int16_t *c = G.at<int16_t>(ws, img, G.o_coef) + (size_t)b * 64;
    int last = 0;
    while (mask) {
        const int z = __ffsll((long long)mask) - 1;
        mask &= mask - 1;
        int run = z - last - 1;
        for (; run > 15; run -= 16) W.code(tabs.ac[t][0xF0]);
        const int v = c[z];
        n = category(v);
        W.code(tabs.ac[t][run << 4 | n]);
        W.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
        last = z;
    }
    if (last != 63) W.code(tabs.ac[t][0]);
    if (b + 1 == G.nblk && info->pad) W.put((1u << info->pad) - 1, (int)info->pad);  // flush_bits
    W.finish();
}

__device__ __forceinline__ uint32_t ent_byte(uint32_t word, int j) { return word >> (24 - 8 * j) & 0xff; }

// the entropy word of this thread and how many of its bytes are data (0..4)
__device__ __forceinline__ uint32_t tile_word(const uint32_t *ent, uint64_t E, uint32_t tile, int &nbytes) {
    const uint64_t wi = (uint64_t)tile * kTileThreads + threadIdx.x;
    const int64_t left = (int64_t)E - 4 * (int64_t)wi;
    nbytes = left <= 0 ? 0 : left >= 4 ? 4 : (int)left;
    return nbytes ? ent[wi] : 0;
}

__device__ __forceinline__ uint32_t count_ff(uint32_t word, int nbytes) {
    uint32_t c = 0;
    for (int j = 0; j < nbytes; ++j) c += ent_byte(word, j) == 0xff;
    return c;
}

__global__ void __launch_bounds__(kTileThreads) k_ff_count(uint8_t *ws, Geo G) {
    const int img = blockIdx.y;
    const uint32_t tile = blockIdx.x;
    const ImgInfo *info = G.at<ImgInfo>(ws, img, G.o_info);
    if (info->error || tile >= info->tiles) return;
    int nb;
    const uint32_t word = tile_word(G.at<uint32_t>(ws, img, G.o_ent), info->bits / 8, tile, nb);
    __shared__ uint32_t sm[kTileThreads / 32];
    const uint32_t c = block_sum<kTileThreads>(count_ff(word, nb), sm);
    if (threadIdx.x == 0) G.at<uint32_t>(ws, img, G.o_tcnt)[tile] = c;
}

__global__ void __launch_bounds__(1024) k_ff_scan(uint8_t *ws, Geo G, uint32_t hdr_len, uint64_t *lens) {
    const int img = blockIdx.x;
    ImgInfo *info = G.at<ImgInfo>(ws, img, G.o_info);
    if (info->error) return;
    uint32_t *a = G.at<uint32_t>(ws, img, G.o_tcnt);
    const uint32_t T = info->tiles, per = (T + 1023) / 1024, lo = min(T, threadIdx.x * per), hi = min(T, lo + per);
    __shared__ uint32_t sm[32];
    uint32_t sum = 0;
    for (uint32_t i = lo; i < hi; ++i) sum += a[i];
    uint32_t total;
    uint32_t run = block_scan<1024>(sum, total, sm);
    for (uint32_t i = lo; i < hi; ++i) {
        const uint32_t v = a[i];
        a[i] = run;
        run += v;
    }
    if (threadIdx.x == 0) {
        const uint64_t len = hdr_len + info->bits / 8 + total + 2;
        lens[img] = len;
        info->ff = total;
        if (len > G.cap) info->error = 2;
    }
}

__global__ void __launch_bounds__(kTileThreads) k_scatter(uint8_t *ws, Geo G, Header hd, uint8_t *files, size_t file_cap) {
    const int img = blockIdx.y;
    const uint32_t tile = blockIdx.x;
    const ImgInfo *info = G.at<ImgInfo>(ws, img, G.o_info);
    if (info->error || tile >= info->tiles) return;
    uint8_t *file = files + (size_t)img * file_cap;
    if (tile == 0)
        for (uint32_t i = threadIdx.x; i < hd.len; i += kTileThreads) file[i] = hd.b[i];
    const uint64_t E = info->bits / 8;
    int nb;
    const uint32_t word = tile_word(G.at<uint32_t>(ws, img, G.o_ent), E, tile, nb);
    __shared__ uint32_t sm[kTileThreads / 32];
    uint32_t total;
    const uint32_t before = G.at<uint32_t>(ws, img, G.o_tcnt)[tile] + block_scan<kTileThreads>(count_ff(word, nb), total, sm);
    uint64_t pos = hd.len + 4 * ((uint64_t)tile * kTileThreads + threadIdx.x) + before;
    for (int j = 0; j < nb; ++j) {
        const uint32_t v = ent_byte(word, j);
        file[pos++] = (uint8_t)v;
        if (v == 0xff) file[pos++] = 0;
    }
    if (tile + 1 == info->tiles && threadIdx.x == 0) {
        const uint64_t end = hd.len + E + info->ff;
        file[end] = 0xFF;
        file[end + 1] = 0xD9;
    }
}

}  // namespace

int JpegExactEncoder::encode(int n, const JpegSrc &src, int components, int w, int h, int quality, size_t capacity, int slot,
                             cudaStream_t s) {
    if (n <= 0) return 0;
    if (components != 1 && components != 3) throw std::runtime_error("jpeg: 1 or 3 components");
    if (w <= 0 || h <= 0 || w > 65535 || h > 65535) throw std::runtime_error("jpeg: image size out of range");
    if (quality < 1 || quality > 100) throw std::runtime_error("jpeg: quality must be in 1..100");
    if (capacity == 0) throw std::runtime_error("jpeg: zero capacity");
    const Geo G(components, w, h, capacity);
    files_.prepare(slot, n, capacity);
    const int E = (int)std::max<size_t>(1, std::min<size_t>((size_t)n, kWorkspaceBudget / G.bytes));
    ws_.grow((size_t)E * G.bytes);
    int launches = 0;
    for (int i0 = 0; i0 < n; i0 += E) {
        JpegSrc part = src;
        part.base = src.base + (size_t)i0 * src.img_stride;
        launches += encode_part(std::min(E, n - i0), part, components, w, h, quality, capacity, files_.file(slot, i0),
                                files_.lens(slot) + i0, s);
    }
    files_.read_lens(slot, n, s);
    return launches;
}

int JpegExactEncoder::encode_part(int n, const JpegSrc &src, int components, int w, int h, int quality, size_t capacity, uint8_t *files,
                                  uint64_t *lens, cudaStream_t s) {
    const Geo G(components, w, h, capacity);
    const QuantTabs Q = make_quant(quality);
    const Header hd = make_header(w, h, components, quality);
    const unsigned nb = (unsigned)ceil_div((int)G.nblk, kBlkThreads);
    k_dct<<<dim3(nb, n), kBlkThreads, 0, s>>>(src, ws_, G, Q);
    DFB_KERNEL_CHECK();
    k_dc<<<dim3(nb, n), kBlkThreads, 0, s>>>(ws_, G);
    DFB_KERNEL_CHECK();
    k_bits<<<n, 1024, 0, s>>>(ws_, G, hd.len, lens);
    DFB_KERNEL_CHECK();
    k_offsets<<<dim3(nb, n), kBlkThreads, 0, s>>>(ws_, G);
    DFB_KERNEL_CHECK();
    k_emit<<<dim3(nb, n), kBlkThreads, 0, s>>>(ws_, G);
    DFB_KERNEL_CHECK();
    k_ff_count<<<dim3(G.tiles_max, n), kTileThreads, 0, s>>>(ws_, G);
    DFB_KERNEL_CHECK();
    k_ff_scan<<<n, 1024, 0, s>>>(ws_, G, hd.len, lens);
    DFB_KERNEL_CHECK();
    k_scatter<<<dim3(G.tiles_max, n), kTileThreads, 0, s>>>(ws_, G, hd, files, capacity);
    DFB_KERNEL_CHECK();
    return 8;
}

size_t JpegExactEncoder::needed(uint64_t reported, const JpegSrc &src, int i, int components, int w, int h, int quality, cudaStream_t s) {
    if (!(reported & kJpegLenLowerBound)) return (size_t)reported;
    // the stuffed zeros at most double the entropy data: encode image i alone with room for that, in the probe's own
    // workspace and files (this encoder's may still be in use by a later group's encode on another stream)
    JpegSrc one = src;
    one.base = src.base + (size_t)i * src.img_stride;
    if (!probe_) probe_.reset(new JpegExactEncoder());
    probe_->encode(1, one, components, w, h, quality, 2 * (size_t)(reported & ~kJpegLenLowerBound), 0, s);
    DFB_CUDA(cudaStreamSynchronize(s));
    return (size_t)probe_->files().host_len(0, 0);
}

}  // namespace dfb
