// jpeg_decode.cu — batched JPEG decode, exactly the pixels of cv2.imdecode(buf, IMREAD_COLOR) (libjpeg-turbo 3.1 with
// OpenCV's settings: JDCT_ISLOW, fancy upsampling, YCbCr -> BGR), for the `-if` frame folders of the reference's decode
// stage (imread(path, IMREAD_COLOR) + cvtColor(BGR2GRAY)).  Integer arithmetic only, so both builds give the same bytes.
//
// Pipeline of one call (n files):
//   host      parse the markers of every file into a descriptor (geometry, quantisation tables, canonical Huffman tables
//             as a 9-bit lookup plus maxcode / valoff for longer codes, restart interval), one H2D of descriptors and the
//             entropy-coded bytes of every file
//   k_destuff one CTA per file: find the marker that ends the scan, drop the 0x00 after each 0xFF, cut the data at its
//             RST markers (checking RST0..7 cycle and count) into segments; 16-byte tiles per thread, counts scanned
//             over the CTA.  Each segment is split into subsequences of kSubBits bits
//   entropy   self-synchronising decode (Klein & Wiseman 2003; Weissenberger & Schmidt 2018 / 2021).  The decoder state
//             is (bit position, block within the MCU, zig-zag index).  Thread t decodes subsequence t from its recorded
//             start state up to the first symbol boundary in subsequence t + 1 and records that state as t + 1's.  The
//             first subsequence of a segment starts from the true state, every other one from a guess; rounds repeat
//             until no record changes (the records then equal the sequential decode's, by induction over t).  A scan of
//             the blocks each subsequence completes gives block indices; a final pass writes de-zig-zagged coefficients
//             and DC differences, and two more scans turn the differences into absolute DC per component and segment.
//   k_idct    jpeg_idct_islow per block into component planes padded to whole MCUs; refuses dequantised values past
//             kMaxDequant (the most an 8-bit encoder writes) and outputs past -512..511
//   errors    a frame's status holds, per restart interval, the first error in decode order (an invalid code whose 16-bit
//             look-ahead runs past the interval's end counts as the interval ending early); the message ranks RST number,
//             RST count, invalid code, early end, no marker after the data, then out-of-range coefficients
//   k_color   one thread per 2 x 2 output block: libjpeg's upsampling (fancy h2v1 / h1v2 / h2v2, box when the chroma
//             plane is at most 2 samples wide for the h2 cases), ycc_rgb_convert, written as BGR, or as BGR2GRAY of it.
#include <cstring>
#include <string>

#include "jpeg_decode.h"

namespace dfb {

namespace {

constexpr int kSubBits = 1024;  // bits per subsequence of the entropy decode
constexpr int kWarmup = 8;      // subsequences decoded from a guess before a start state is first recorded
constexpr int kDT = 512;        // threads of k_destuff
constexpr int kDB = 16;         // bytes per thread and tile of k_destuff

enum : int { kErrCode = 1, kErrShort = 2, kErrRst = 4, kErrRstCount = 8, kErrRange = 16, kErrNoEnd = 32 };

// The largest |coefficient x quantisation value| libjpeg's islow forward DCT and quantiser produce from 8-bit samples at any
// table entry (DESIGN §7).  Past it imdecode's pixels depend on how libjpeg-turbo was built, so the file is refused.
constexpr int kMaxDequant = 2048;

struct HuffTab {
    uint16_t fast[512];  // 9-bit look-ahead -> (length << 8) | symbol, length 0: a longer code
    int32_t maxcode[17];
    int32_t valoff[17];
    uint8_t vals[256];
};

struct JFrame {
    int w, h, ncomp, bpm, mcux, mcuy, hmax, vmax;
    int ri, nseg, seg_base;
    int raw_len;
    long long raw_off, blk_base;
    int sub_base, sub_bound;
    int lay_ci[6], lay_bx[6], lay_by[6];
    int ch[3], cv[3], dc[3], ac[3], q[3];
    int cw[3], chh[3];  // downsampled_width / downsampled_height of each component
    long long plane_off[3];
    int plane_pitch[3];
};

// exclusive scan over the CTA (NT threads); total receives the sum.  sm: 32 words.
template <int NT> __device__ int cta_scan(int v, int &total, int *sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sm[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int t = lane < NT / 32 ? sm[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        if (lane < NT / 32) sm[lane] = t;
    }
    __syncthreads();
    const int base = warp ? sm[warp - 1] : 0;
    total = sm[NT / 32 - 1];
    __syncthreads();
    return base + x - v;
}

__global__ void __launch_bounds__(kDT) k_destuff(const uint8_t *__restrict__ raw, uint8_t *__restrict__ ds, const JFrame *__restrict__ F,
                                                 int *seg_start, int *seg_bytes, int *seg_sub_base, int *seg_nsub, int *status) {
    __shared__ int sm[32];
    __shared__ int s_end;
    const JFrame &f = F[blockIdx.x];
    const uint8_t *r = raw + f.raw_off;
    const int L = f.raw_len;
    if (threadIdx.x == 0) s_end = L;
    __syncthreads();
    // the scan ends at the first marker that is neither a stuffed zero nor RSTn (EOI, or anything after the data)
    for (int j = threadIdx.x + 1; j < L; j += kDT)
        if (r[j - 1] == 0xFF) {
            const int b = r[j];
            if (b != 0 && b != 0xFF && (b < 0xD0 || b > 0xD7)) atomicMin(&s_end, j - 1);
        }
    __syncthreads();
    const int end = s_end;
    int carry = 0, rcarry = 0, bad = 0;
    for (int base = 0; base < end; base += kDT * kDB) {
        const int j0 = base + threadIdx.x * kDB;
        uint32_t keep = 0, rst = 0;
        for (int i = 0; i < kDB && j0 + i < end; ++i) {
            const int j = j0 + i, b = r[j];
            if (b == 0xFF) {
                if (j + 1 < L && r[j + 1] == 0) keep |= 1u << i;  // a data byte 0xFF; fill bytes and marker prefixes go
            } else if (j > 0 && r[j - 1] == 0xFF) {
                if (b >= 0xD0 && b <= 0xD7) rst |= 1u << i;  // the stuffed zero and marker codes go
            } else {
                keep |= 1u << i;
            }
        }
        int tk, tr;
        int o = carry + cta_scan<kDT>(__popc(keep), tk, sm);
        int ri = rcarry + cta_scan<kDT>(__popc(rst), tr, sm);
        for (int i = 0; i < kDB; ++i) {
            if ((keep >> i) & 1) {
                ds[f.raw_off + o++] = r[j0 + i];
            } else if ((rst >> i) & 1) {
                if (r[j0 + i] - 0xD0 != (ri & 7)) bad |= kErrRst;
                if (ri + 1 < f.nseg) seg_start[f.seg_base + ri + 1] = o;
                ++ri;
            }
        }
        carry += tk;
        rcarry += tr;
    }
    if (rcarry != f.nseg - 1) bad |= kErrRstCount;
    if (bad) atomicOr(&status[blockIdx.x], bad);
    if (end == L && threadIdx.x == 0) atomicOr(&status[blockIdx.x], kErrNoEnd);  // no marker after the data; it still decodes
    const bool fbad = __syncthreads_or(bad != 0);
    // segments and their subsequences; a frame with a bad marker sequence decodes nothing (its status is already set)
    int sub_carry = 0;
    for (int s0 = 0; s0 < f.nseg; s0 += kDT) {
        const int s = s0 + threadIdx.x;
        int nsub = 0, bytes = 0;
        if (s < f.nseg) {
            if (!fbad) {
                const int st = s ? seg_start[f.seg_base + s] : 0;
                bytes = (s + 1 < f.nseg ? seg_start[f.seg_base + s + 1] : carry) - st;
            }
            nsub = max(1, ceil_div(bytes * 8, kSubBits));
        }
        int tot;
        const int off = cta_scan<kDT>(nsub, tot, sm);
        if (s < f.nseg) {
            const int g = f.seg_base + s;
            if (fbad || s == 0) seg_start[g] = 0;
            seg_bytes[g] = bytes;
            seg_nsub[g] = nsub;
            seg_sub_base[g] = f.sub_base + sub_carry + off;
        }
        sub_carry += tot;
        __syncthreads();
    }
}

// 32 bits of the de-stuffed stream from bit P on (the buffer is 4-byte aligned and padded past every frame's data)
__device__ __forceinline__ uint32_t peek32(const uint8_t *ds, uint64_t P) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(ds) + (P >> 5);
    const uint64_t v = ((uint64_t)__byte_perm(__ldg(w), 0, 0x0123) << 32) | __byte_perm(__ldg(w + 1), 0, 0x0123);
    return (uint32_t)((v << (P & 31)) >> 32);
}

__device__ __forceinline__ uint64_t pack_state(uint32_t pos, int zz, int blk) {
    return (uint64_t)pos | ((uint64_t)zz << 32) | ((uint64_t)blk << 40);
}

__constant__ uint8_t c_natural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
    6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
    39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

enum : int { kRunEnd = 0, kRunOverrun = 1, kRunBadCode = 2, kRunBlocksDone = 3 };

struct Run {
    uint32_t pos;
    int zz, blk, done, ndc;
    int dcsum[3];
};

// Decodes symbols from the state in R until the position reaches end_bit (the state then is the first symbol boundary at or
// after it), a symbol would need bits past seg_bits, a code is invalid, or (WRITE) max_blocks blocks are complete.
// WRITE: coefficients of block `first_block + done` go to coef (AC in natural order, the DC difference at [0]).
template <bool WRITE>
__device__ int run_decode(const uint8_t *ds, uint64_t seg_bit0, uint32_t seg_bits, uint32_t end_bit, const JFrame &f,
                          const HuffTab *__restrict__ tabs, Run &R, int16_t *coef, long long first_block, int max_blocks) {
    while (R.pos < end_bit) {
        if (WRITE && R.done >= max_blocks) return kRunBlocksDone;
        const int ci = f.lay_ci[R.blk];
        const HuffTab &T = tabs[R.zz == 0 ? f.dc[ci] : f.ac[ci]];
        const uint32_t bits = peek32(ds, seg_bit0 + R.pos);
        const uint32_t b16 = bits >> 16;
        int len = 0, sym = 0;
        const uint32_t e = __ldg(&T.fast[b16 >> 7]);
        if (e >> 8) {
            len = e >> 8;
            sym = e & 255;
        } else {
            for (int l = 10; l <= 16; ++l) {
                const int code = (int)(b16 >> (16 - l));
                if (code <= __ldg(&T.maxcode[l])) {
                    len = l;
                    sym = __ldg(&T.vals[code + __ldg(&T.valoff[l])]);
                    break;
                }
            }
            // a code that matches nothing only because of bits past the segment's end is the segment ending early
            if (!len) return R.pos + 16 > seg_bits ? kRunOverrun : kRunBadCode;
        }
        const int nb = R.zz == 0 ? sym : (sym & 15);
        if (R.pos + len + nb > seg_bits) return kRunOverrun;
        int val = 0;
        if (nb) {
            const int v = (int)((bits << len) >> (32 - nb));
            val = v < (1 << (nb - 1)) ? v - (1 << nb) + 1 : v;  // HUFF_EXTEND
        }
        R.pos += len + nb;
        int16_t *blk = WRITE ? coef + (first_block + R.done) * 64 : nullptr;
        if (R.zz == 0) {
            if (WRITE) {
                blk[0] = (int16_t)val;
                R.dcsum[ci] += val;
                ++R.ndc;
            }
            R.zz = 1;
        } else if (sym & 15) {
            R.zz += sym >> 4;
            if (WRITE) blk[c_natural[R.zz]] = (int16_t)val;
            ++R.zz;
        } else if ((sym >> 4) == 15) {
            R.zz += 16;
        } else {
            R.zz = 64;  // EOB
        }
        if (R.zz >= 64) {
            R.zz = 0;
            R.blk = R.blk + 1 == f.bpm ? 0 : R.blk + 1;
            ++R.done;
        }
    }
    return kRunEnd;
}

struct SubCtx {
    int s, k, nsub, frame;
    uint32_t seg_bits;
    uint64_t seg_bit0;
};

__device__ __forceinline__ bool sub_ctx(int t, const int *sub_seg, const int *seg_sub_base, const int *seg_nsub, const int *seg_start,
                                        const int *seg_bytes, const int *seg_frame, const JFrame *F, SubCtx &c) {
    c.s = sub_seg[t];
    if (c.s < 0) return false;
    c.k = t - seg_sub_base[c.s];
    c.nsub = seg_nsub[c.s];
    c.frame = seg_frame[c.s];
    c.seg_bits = (uint32_t)seg_bytes[c.s] * 8u;
    c.seg_bit0 = ((uint64_t)F[c.frame].raw_off + (uint64_t)seg_start[c.s]) * 8u;
    return true;
}

struct EntropyArgs {
    const uint8_t *ds;
    const JFrame *F;
    const HuffTab *tabs;
    int *sub_seg;
    const int *seg_sub_base, *seg_nsub, *seg_start, *seg_bytes, *seg_frame, *seg_nblocks;
    const long long *seg_first_block;
    uint64_t *st;
    int *cnt, *ndc, *dcsum, *dcbase, *err;
    long long *blk_off, *first_dc;
    int16_t *coef;
    int *status;
    int n_sub, n;
};

// The segment of every subsequence slot (-1: past its frame's data) and its first start state.  Subsequence k of a segment
// decodes the kWarmup subsequences before it from a guess (their first bit, block 0, zig-zag index 0), or from the true
// state when k <= kWarmup, and records where that decode enters subsequence k.  With several blocks per MCU the decoder
// needs more than one subsequence to fall into step (bit position, block and zig-zag index all equal the true decode's),
// so a warm-up of this length leaves few records for the rounds to fix.
__global__ void __launch_bounds__(128) k_init_states(EntropyArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_sub) return;
    int lo = 0, hi = a.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.F[mid].sub_base <= t) lo = mid; else hi = mid - 1;
    }
    const JFrame &f = a.F[lo];
    int g0 = f.seg_base, g1 = f.seg_base + f.nseg - 1;
    while (g0 < g1) {
        const int mid = (g0 + g1 + 1) >> 1;
        if (a.seg_sub_base[mid] <= t) g0 = mid; else g1 = mid - 1;
    }
    const int k = t - a.seg_sub_base[g0];
    if (k >= a.seg_nsub[g0]) {
        a.sub_seg[t] = -1;
        return;
    }
    a.sub_seg[t] = g0;
    uint64_t st = pack_state((uint32_t)k * kSubBits, 0, 0);
    if (k > 0) {
        const int k0 = max(k - kWarmup, 0);
        Run R{(uint32_t)k0 * kSubBits, 0, 0, 0, 0, {0, 0, 0}};
        const uint64_t bit0 = ((uint64_t)f.raw_off + (uint64_t)a.seg_start[g0]) * 8u;
        if (run_decode<false>(a.ds, bit0, (uint32_t)a.seg_bytes[g0] * 8u, (uint32_t)k * kSubBits, f, a.tabs, R, nullptr, 0, 0) == kRunEnd)
            st = pack_state(R.pos, R.zz, R.blk);
    }
    a.st[t] = st;
}

// one round: every subsequence re-decodes from its record and updates its successor's
__global__ void __launch_bounds__(128) k_sync_round(EntropyArgs a, int *changed) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_sub) return;
    SubCtx c;
    if (!sub_ctx(t, a.sub_seg, a.seg_sub_base, a.seg_nsub, a.seg_start, a.seg_bytes, a.seg_frame, a.F, c) || c.k + 1 >= c.nsub) return;
    const JFrame &f = a.F[c.frame];
    const uint64_t s0 = a.st[t];
    Run R{(uint32_t)s0, (int)(s0 >> 32) & 255, (int)(s0 >> 40) & 255, 0, 0, {0, 0, 0}};
    const int rc = run_decode<false>(a.ds, c.seg_bit0, c.seg_bits, (uint32_t)(c.k + 1) * kSubBits, f, a.tabs, R, nullptr, 0, 0);
    // a subsequence that meets an invalid code or the end of the segment hands its successor the initial guess; only a
    // record reached from the true state matters, and the final pass reports the error there
    const uint64_t next = rc == kRunEnd ? pack_state(R.pos, R.zz, R.blk) : pack_state((uint32_t)(c.k + 1) * kSubBits, 0, 0);
    a.cnt[t] = R.done;
    if (a.st[t + 1] != next) {
        a.st[t + 1] = next;
        *changed = 1;
    }
}

// one warp per segment: exclusive scans over its subsequences.  mode 0: block index of each subsequence's first block (from
// the blocks the subsequences complete); mode 1: the DC predictor of each component at each subsequence's start, and the
// segment's first error in decode order goes to its frame's status (a subsequence after it started from a guess).
__global__ void __launch_bounds__(128) k_seg_scan(EntropyArgs a, int n_seg, int mode) {
    const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= n_seg) return;
    const int b = a.seg_sub_base[s], n = a.seg_nsub[s];
    long long carry[3] = {mode ? 0 : a.seg_first_block[s], 0, 0};
    for (int k0 = 0; k0 < n; k0 += 32) {
        const int k = k0 + lane;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (mode == 0 && c) break;
            long long v = k < n ? (mode ? (long long)a.dcsum[(size_t)(b + k) * 3 + c] : (long long)(k + 1 < n ? a.cnt[b + k] : 0)) : 0;
            long long x = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (k < n) {
                if (mode)
                    a.dcbase[(size_t)(b + k) * 3 + c] = (int)(carry[c] + x - v);
                else
                    a.blk_off[b + k] = carry[c] + x - v;
            }
            carry[c] += __shfl_sync(0xffffffffu, x, 31);
        }
        if (mode) {
            const unsigned m = __ballot_sync(0xffffffffu, k < n && a.err[b + k] != 0);
            if (m) {
                if (lane == __ffs(m) - 1) atomicOr(&a.status[a.seg_frame[s]], a.err[b + k]);
                break;
            }
        }
    }
}

// final pass from the converged records: coefficients, DC differences, errors
__global__ void __launch_bounds__(128) k_decode_final(EntropyArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_sub) return;
    SubCtx c;
    if (!sub_ctx(t, a.sub_seg, a.seg_sub_base, a.seg_nsub, a.seg_start, a.seg_bytes, a.seg_frame, a.F, c)) return;
    const JFrame &f = a.F[c.frame];
    const uint64_t s0 = a.st[t];
    Run R{(uint32_t)s0, (int)(s0 >> 32) & 255, (int)(s0 >> 40) & 255, 0, 0, {0, 0, 0}};
    const long long first = a.blk_off[t], seg_end = a.seg_first_block[c.s] + a.seg_nblocks[c.s];
    const int max_blocks = (int)max(seg_end - first, 0LL);
    const bool last = c.k + 1 == c.nsub;
    a.first_dc[t] = first + (R.zz > 0 ? 1 : 0);
    const int rc = run_decode<true>(a.ds, c.seg_bit0, c.seg_bits, last ? c.seg_bits : (uint32_t)(c.k + 1) * kSubBits, f, a.tabs, R,
                                    a.coef, first, max_blocks);
    a.ndc[t] = R.ndc;
#pragma unroll
    for (int i = 0; i < 3; ++i) a.dcsum[(size_t)t * 3 + i] = R.dcsum[i];
    a.err[t] = rc == kRunBadCode                                                                 ? kErrCode
               : rc != kRunBlocksDone && R.done < max_blocks && (last || rc == kRunOverrun) ? kErrShort
                                                                                            : 0;
}

// absolute DC: each subsequence adds its components' predictors to the differences it decoded
__global__ void __launch_bounds__(128) k_dc_fix(EntropyArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_sub) return;
    const int s = a.sub_seg[t];
    if (s < 0) return;
    const JFrame &f = a.F[a.seg_frame[s]];
    int pred[3] = {a.dcbase[(size_t)t * 3], a.dcbase[(size_t)t * 3 + 1], a.dcbase[(size_t)t * 3 + 2]};
    const long long b0 = a.first_dc[t], seg0 = a.seg_first_block[s];
    for (int i = 0; i < a.ndc[t]; ++i) {
        const long long b = b0 + i;
        const int ci = f.lay_ci[(int)((b - seg0) % f.bpm)];
        pred[ci] += a.coef[b * 64];
        a.coef[b * 64] = (int16_t)pred[ci];
    }
}

// jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) of one 8-point column / row.  T: int for the columns (inputs within
// kMaxDequant + 1 stay far from overflow), long long for the rows (a damaged block's columns can reach ~2^16, whose
// products pass 2^31)
template <typename T> struct Idct8 {
    T o[8];
    __device__ __forceinline__ Idct8(T c0, T c1, T c2, T c3, T c4, T c5, T c6, T c7) {
        T z1 = (c2 + c6) * 4433;
        const T tmp2 = z1 + c6 * -15137, tmp3 = z1 + c2 * 6270;
        const T tmp0 = (c0 + c4) * 8192, tmp1 = (c0 - c4) * 8192;
        const T t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
        T o0 = c7, o1 = c5, o2 = c3, o3 = c1;
        z1 = o0 + o3;
        T z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
        const T z5 = (z3 + z4) * 9633;
        o0 *= 2446;
        o1 *= 16819;
        o2 *= 25172;
        o3 *= 12299;
        z1 *= -7373;
        z2 *= -20995;
        z3 = z3 * -16069 + z5;
        z4 = z4 * -3196 + z5;
        o0 += z1 + z3;
        o1 += z2 + z4;
        o2 += z2 + z3;
        o3 += z1 + z4;
        o[0] = t10 + o3;
        o[7] = t10 - o3;
        o[1] = t11 + o2;
        o[6] = t11 - o2;
        o[2] = t12 + o1;
        o[5] = t12 - o1;
        o[3] = t13 + o0;
        o[4] = t13 - o0;
    }
};

__device__ __forceinline__ int find_frame(const JFrame *F, int n, long long b) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (F[mid].blk_base <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// one thread per block: dequantise, inverse DCT, range limit (the post-IDCT table of jdmaster.c: the value masked to 10 bits
// as a signed number, + 128, clamped), into the component plane.  A dequantised value past kMaxDequant, or an output past
// -512..511 (where the table wraps and libjpeg-turbo's SIMD IDCT saturates instead), sets kErrRange; the IDCT runs on
// values clamped to kMaxDequant + 1, so it cannot overflow (the frame is refused anyway).
__global__ void __launch_bounds__(128) k_idct(const int16_t *__restrict__ coef, const JFrame *__restrict__ F, int n, long long n_blocks,
                                              const int32_t *__restrict__ quant, uint8_t *__restrict__ planes, int *status) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const int fi = find_frame(F, n, b);
    const JFrame &f = F[fi];
    const long long lb = b - f.blk_base;
    const int mcu = (int)(lb / f.bpm), k = (int)(lb % f.bpm);
    const int ci = f.lay_ci[k];
    const int bx = (mcu % f.mcux) * f.ch[ci] + f.lay_bx[k], by = (mcu / f.mcux) * f.cv[ci] + f.lay_by[k];
    const int32_t *q = quant + (size_t)(fi * 4 + f.q[ci]) * 64;
    int c[64];
    bool out_of_range = false;
    const int4 *src = reinterpret_cast<const int4 *>(coef + b * 64);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int4 v = __ldg(src + i);
        const int w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int d = (int)(int16_t)(h ? (uint32_t)w4[j] >> 16 : w4[j] & 0xFFFF) * __ldg(q + i * 8 + 2 * j + h);
                out_of_range |= d > kMaxDequant || d < -kMaxDequant;
                c[i * 8 + 2 * j + h] = min(max(d, -kMaxDequant - 1), kMaxDequant + 1);
            }
        }
    }
    int ws[64];
#pragma unroll
    for (int x = 0; x < 8; ++x) {  // pass 1: columns
        const Idct8<int> d(c[x], c[8 + x], c[16 + x], c[24 + x], c[32 + x], c[40 + x], c[48 + x], c[56 + x]);
#pragma unroll
        for (int y = 0; y < 8; ++y) ws[y * 8 + x] = (d.o[y] + (1 << 10)) >> 11;
    }
    uint8_t *dst = planes + f.plane_off[ci] + (size_t)(by * 8) * f.plane_pitch[ci] + bx * 8;
#pragma unroll
    for (int y = 0; y < 8; ++y) {  // pass 2: rows
        const Idct8<long long> d(ws[y * 8], ws[y * 8 + 1], ws[y * 8 + 2], ws[y * 8 + 3], ws[y * 8 + 4], ws[y * 8 + 5], ws[y * 8 + 6],
                                 ws[y * 8 + 7]);
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int x = 0; x < 8; ++x) {
            const long long v64 = (d.o[x] + (1 << 17)) >> 18;
            out_of_range |= v64 < -512 || v64 > 511;
            const int v = (int)v64;
            const int s = ((v & 1023) ^ 512) - 512;
            const uint32_t px = (uint32_t)min(max(s + 128, 0), 255);
            if (x < 4) lo |= px << (8 * x); else hi |= px << (8 * (x - 4));
        }
        *reinterpret_cast<uint2 *>(dst + (size_t)y * f.plane_pitch[ci]) = make_uint2(lo, hi);
    }
    if (out_of_range) atomicOr(&status[fi], kErrRange);
}

// libjpeg's upsampled chroma sample at output (x, y) of a plane of cw x ch samples (fh, fv: 1 or 2)
__device__ __forceinline__ int chroma_at(const uint8_t *__restrict__ P, int pitch, int cw, int ch, int fh, int fv, int x, int y) {
    if (fv == 1) {
        const uint8_t *r = P + (size_t)y * pitch;
        if (fh == 1) return r[x];
        const int i = x >> 1;  // h2v1_fancy_upsample / h2v1_upsample
        if (cw <= 2) return r[i];
        if (x & 1) return i == cw - 1 ? r[i] : (3 * r[i] + r[i + 1] + 2) >> 2;
        return i == 0 ? r[0] : (3 * r[i] + r[i - 1] + 1) >> 2;
    }
    const int j = y >> 1, nb = (y & 1) ? min(j + 1, ch - 1) : max(j - 1, 0);
    const uint8_t *r0 = P + (size_t)j * pitch, *r1 = P + (size_t)nb * pitch;
    if (fh == 1) return (3 * r0[x] + r1[x] + ((y & 1) ? 2 : 1)) >> 2;  // h1v2_fancy_upsample
    const int i = x >> 1;
    if (cw <= 2) return r0[i];  // h2v2_upsample
    const int cs = 3 * r0[i] + r1[i];  // h2v2_fancy_upsample
    if (x & 1) return i == cw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * r0[i + 1] + r1[i + 1] + 7) >> 4;
    return i == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * r0[i - 1] + r1[i - 1] + 8) >> 4;
}

// one thread per 2 x 2 output block of frame blockIdx.z
__global__ void __launch_bounds__(256) k_color(const JFrame *__restrict__ F, const uint8_t *__restrict__ planes, int channels,
                                               uint8_t *__restrict__ out, size_t pitch, size_t frame_stride) {
    const JFrame &f = F[blockIdx.z];
    const int cx = blockIdx.x * 32 + threadIdx.x, cy = blockIdx.y * 8 + threadIdx.y;
    if (2 * cx >= f.w || 2 * cy >= f.h) return;
    uint8_t *o = out + frame_stride * blockIdx.z;
    const uint8_t *Y = planes + f.plane_off[0];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int y = 2 * cy + j;
        if (y >= f.h) break;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int x = 2 * cx + i;
            if (x >= f.w) break;
            const int yy = Y[(size_t)y * f.plane_pitch[0] + x];
            int b = yy, g = yy, r = yy;
            if (f.ncomp == 3) {  // ycc_rgb_convert (jdcolor.c), SCALEBITS 16
                const int fh = f.hmax / f.ch[1], fv = f.vmax / f.cv[1];
                const int cb = chroma_at(planes + f.plane_off[1], f.plane_pitch[1], f.cw[1], f.chh[1], fh, fv, x, y) - 128;
                const int cr = chroma_at(planes + f.plane_off[2], f.plane_pitch[2], f.cw[2], f.chh[2], fh, fv, x, y) - 128;
                r = min(max(yy + ((91881 * cr + 32768) >> 16), 0), 255);
                g = min(max(yy + ((-46802 * cr + (-22554 * cb + 32768)) >> 16), 0), 255);
                b = min(max(yy + ((116130 * cb + 32768) >> 16), 0), 255);
            }
            if (channels == 1) {
                o[(size_t)y * pitch + x] = (uint8_t)((b * 3735 + g * 19235 + r * 9798 + 16384) >> 15);  // cvtColor(BGR2GRAY)
            } else {
                uint8_t *p = o + (size_t)y * pitch + 3 * x;
                p[0] = (uint8_t)b;
                p[1] = (uint8_t)g;
                p[2] = (uint8_t)r;
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------

const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

[[noreturn]] void corrupt(int index, const std::string &m) { throw std::runtime_error("frame " + std::to_string(index) + ": " + m); }
[[noreturn]] void unsupported(int index, const std::string &m) { throw JpegUnsupported("frame " + std::to_string(index) + ": " + m); }

int u16(const uint8_t *p) { return (p[0] << 8) | p[1]; }

// Orientation tag (0x0112) of IFD0 of an APP1 Exif payload, or 1
int exif_orientation(const uint8_t *p, size_t n) {
    if (n < 14 || std::memcmp(p, "Exif\0\0", 6) != 0) return 1;
    const uint8_t *t = p + 6;
    const size_t tn = n - 6;
    bool le;
    if (t[0] == 'I' && t[1] == 'I') le = true;
    else if (t[0] == 'M' && t[1] == 'M') le = false;
    else return 1;
    auto rd = [&](size_t o, int k) -> uint32_t {
        uint32_t v = 0;
        for (int i = 0; i < k; ++i) v |= (uint32_t)t[o + i] << (8 * (le ? i : k - 1 - i));
        return v;
    };
    const size_t ifd = rd(4, 4);
    if (ifd + 2 > tn) return 1;
    const int ne = (int)rd(ifd, 2);
    for (int e = 0; e < ne; ++e) {
        const size_t o = ifd + 2 + 12 * (size_t)e;
        if (o + 12 > tn) break;
        if (rd(o, 2) == 0x0112) return (int)rd(o + 8, 2);
    }
    return 1;
}

const char *sof_name(int m) {
    switch (m) {
    case 0xC2: return "progressive";
    case 0xC3: return "lossless";
    case 0xC5: return "differential sequential";
    case 0xC6: return "differential progressive";
    case 0xC7: return "differential lossless";
    case 0xC9: return "arithmetic-coded";
    case 0xCA: return "arithmetic-coded progressive";
    case 0xCB: return "arithmetic-coded lossless";
    case 0xCD: case 0xCE: case 0xCF: return "arithmetic-coded differential";
    default: return nullptr;
    }
}

void build_table(const JpegHeader::Table &t, HuffTab &o) {
    std::memset(&o, 0, sizeof(o));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        o.valoff[l] = k - code;
        for (int i = 0; i < t.counts[l - 1]; ++i, ++k, ++code) {
            o.vals[k] = t.symbols[k];
            if (l <= 9)
                for (int fill = 0; fill < (1 << (9 - l)); ++fill) o.fast[(code << (9 - l)) | fill] = (uint16_t)((l << 8) | t.symbols[k]);
        }
        o.maxcode[l] = t.counts[l - 1] ? code - 1 : -1;
        code <<= 1;
    }
}

}  // namespace

JpegHeader parse_jpeg_header(const uint8_t *b, size_t len, int index) {
    JpegHeader hd;
    if (len < 4 || b[0] != 0xFF || b[1] != 0xD8) corrupt(index, "not a JPEG file (no SOI marker)");
    bool jfif = false, have_sof = false;
    int adobe = -1, orient = 1;
    int comp_id[4] = {}, comp_hv[4] = {}, comp_tq[4] = {};
    size_t i = 2;
    for (;;) {
        if (i < len && b[i] != 0xFF) corrupt(index, "garbage between markers");
        while (i < len && b[i] == 0xFF) ++i;
        if (i + 2 >= len) corrupt(index, "file ends before the scan");
        const int m = b[i++];
        if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) corrupt(index, "unexpected marker before the scan");
        const size_t L = (size_t)u16(b + i);
        if (L < 2 || i + L > len) corrupt(index, "marker segment runs past the end of the file");
        const uint8_t *p = b + i + 2;
        const size_t pn = L - 2;
        i += L;
        if (const char *nm = sof_name(m)) unsupported(index, std::string(nm) + " JPEG (SOF" + std::to_string(m - 0xC0) + ") is not supported");
        if (m == 0xC0 || m == 0xC1) {
            if (pn < 6) corrupt(index, "short frame header");
            if (p[0] != 8) unsupported(index, std::to_string(p[0]) + "-bit samples are not supported (8-bit only)");
            hd.h = u16(p + 1);
            hd.w = u16(p + 3);
            hd.ncomp = p[5];
            if (hd.ncomp == 4) unsupported(index, "CMYK / 4-component JPEG is not supported");
            if (hd.ncomp != 1 && hd.ncomp != 3) unsupported(index, std::to_string(hd.ncomp) + "-component JPEG is not supported");
            if (pn < 6 + 3 * (size_t)hd.ncomp) corrupt(index, "short frame header");
            for (int c = 0; c < hd.ncomp; ++c) {
                comp_id[c] = p[6 + 3 * c];
                comp_hv[c] = p[7 + 3 * c];
                comp_tq[c] = p[8 + 3 * c];
            }
            have_sof = true;
        } else if (m == 0xC4) {
            size_t o = 0;
            while (o < pn) {
                if (o + 17 > pn) corrupt(index, "short DHT segment");
                const int tc = p[o] >> 4, th = p[o] & 15;
                if (tc > 1 || th > 3) corrupt(index, "bad DHT table id");
                JpegHeader::Table &t = tc ? hd.ac[th] : hd.dc[th];
                int total = 0;
                for (int l = 0; l < 16; ++l) total += t.counts[l] = p[o + 1 + l];
                if (total > 256 || o + 17 + total > pn) corrupt(index, "bad Huffman table");
                std::memcpy(t.symbols, p + o + 17, total);
                int code = 0;  // jpeg_make_d_derived_tbl: no code may be all ones
                for (int l = 1; l <= 16; ++l) {
                    code += t.counts[l - 1];
                    if (t.counts[l - 1] && code >= (1 << l)) corrupt(index, "bad Huffman table");
                    code <<= 1;
                }
                if (tc == 0)
                    for (int s = 0; s < total; ++s)
                        if (t.symbols[s] > 15) corrupt(index, "bad Huffman table");
                t.defined = true;
                o += 17 + total;
            }
        } else if (m == 0xDB) {
            size_t o = 0;
            while (o < pn) {
                const int pq = p[o] >> 4, tq = p[o] & 15;
                if (tq > 3) corrupt(index, "bad DQT table id");
                if (o + 1 + 64 * (pq ? 2 : 1) > pn) corrupt(index, "short DQT segment");
                for (int k = 0; k < 64; ++k) {
                    const int v = pq ? u16(p + o + 1 + 2 * k) : p[o + 1 + k];
                    hd.quant[tq][kZigzag[k]] = (int16_t)v;  // ISLOW_MULT_TYPE is 16-bit
                }
                hd.has_quant[tq] = true;
                o += 1 + 64 * (pq ? 2 : 1);
            }
        } else if (m == 0xDD) {
            if (pn < 2) corrupt(index, "short DRI segment");
            hd.ri = u16(p);
        } else if (m == 0xE0) {
            jfif = jfif || (pn >= 5 && std::memcmp(p, "JFIF\0", 5) == 0);
        } else if (m == 0xE1) {
            const int o = exif_orientation(p, pn);
            if (orient == 1) orient = o;
        } else if (m == 0xEE) {
            if (pn >= 12 && std::memcmp(p, "Adobe", 5) == 0) adobe = p[11];
        } else if (m == 0xDA) {
            if (!have_sof) corrupt(index, "scan before the frame header");
            if (pn < 1) corrupt(index, "short scan header");
            const int ns = p[0];
            if (pn < 4 + 2 * (size_t)ns) corrupt(index, "short scan header");
            if (hd.w == 0 || hd.h == 0) unsupported(index, "JPEG without its size in the frame header (DNL) is not supported");
            if (ns != hd.ncomp)
                unsupported(index, "multi-scan JPEG is not supported (the first scan holds " + std::to_string(ns) + " of " +
                                       std::to_string(hd.ncomp) + " components)");
            if (p[1 + 2 * ns] != 0 || p[2 + 2 * ns] != 63 || p[3 + 2 * ns] != 0) corrupt(index, "bad spectral selection in a sequential scan");
            if (hd.ncomp == 3) {
                const bool ids123 = comp_id[0] == 1 && comp_id[1] == 2 && comp_id[2] == 3;
                const bool ycc = jfif || (adobe >= 0 ? adobe == 1 : ids123);
                if (!ycc) unsupported(index, "RGB-coded JPEG is not supported (YCbCr only)");
                const int h0 = comp_hv[0] >> 4, v0 = comp_hv[0] & 15;
                if (comp_hv[1] != 0x11 || comp_hv[2] != 0x11 || h0 < 1 || h0 > 2 || v0 < 1 || v0 > 2) {
                    std::string s;
                    for (int c = 0; c < 3; ++c) s += (c ? "," : "") + std::to_string(comp_hv[c] >> 4) + "x" + std::to_string(comp_hv[c] & 15);
                    unsupported(index, "chroma subsampling " + s + " is not supported (4:4:4, 4:2:2, 4:4:0, 4:2:0 only)");
                }
            }
            if (orient >= 2 && orient <= 8)
                unsupported(index, "EXIF orientation " + std::to_string(orient) + " is not supported (imdecode would rotate the image)");
            for (int k = 0; k < ns; ++k) {
                const int cid = p[1 + 2 * k], td = p[2 + 2 * k] >> 4, ta = p[2 + 2 * k] & 15;
                int c = -1;
                for (int j = 0; j < hd.ncomp; ++j)
                    if (comp_id[j] == cid) c = j;
                if (c < 0 || td > 3 || ta > 3) corrupt(index, "scan component does not match the frame");
                const int tq = comp_tq[c] & 3;
                if (!hd.has_quant[tq] || !hd.dc[td].defined || !hd.ac[ta].defined) corrupt(index, "scan uses an undefined table");
                hd.comp_q[k] = tq;  // a full scan lists the frame's components; k follows the scan order
                hd.comp_dc[k] = td;
                hd.comp_ac[k] = ta;
                hd.comp_h[k] = hd.ncomp == 1 ? 1 : comp_hv[c] >> 4;
                hd.comp_v[k] = hd.ncomp == 1 ? 1 : comp_hv[c] & 15;
            }
            hd.hmax = hd.comp_h[0];
            hd.vmax = hd.comp_v[0];
            if (hd.ncomp == 3 && (hd.comp_h[1] != 1 || hd.comp_v[1] != 1 || hd.comp_h[2] != 1 || hd.comp_v[2] != 1))
                unsupported(index, "a scan that does not start with the luma component is not supported");
            hd.mcux = ceil_div(hd.w, 8 * hd.hmax);
            hd.mcuy = ceil_div(hd.h, 8 * hd.vmax);
            hd.bpm = 0;
            for (int c = 0; c < hd.ncomp; ++c) hd.bpm += hd.comp_h[c] * hd.comp_v[c];
            const long long nmcu = (long long)hd.mcux * hd.mcuy;
            hd.nseg = hd.ri ? (int)((nmcu + hd.ri - 1) / hd.ri) : 1;
            hd.data_off = i;
            return hd;
        }
    }
}

struct JpegDecoder::Layout {
    int n = 0, n_tab = 0, n_seg = 0, n_sub = 0;
    long long n_blocks = 0;
    size_t raw_bytes = 0, plane_bytes = 0;
    // offsets into the workspace; [0, upload) is copied from the staging buffer
    size_t o_frames, o_tabs, o_quant, o_seg_frame, o_seg_first, o_seg_nblocks, o_raw, upload;
    size_t o_ds, o_seg_start, o_seg_bytes, o_seg_sub_base, o_seg_nsub, o_sub_seg, o_st, o_cnt, o_ndc, o_dcsum, o_dcbase, o_err, o_blk_off,
        o_first_dc, o_status, o_flag, o_coef, o_planes, total;
};

JpegDecoder::~JpegDecoder() { delete L; }

static size_t a256(size_t x) { return (x + 255) & ~size_t(255); }

void JpegDecoder::run_entropy(const uint8_t *const *jpeg, const size_t *len, const JpegHeader *hd, int n, cudaStream_t s) {
    if (!L) L = new Layout();
    Layout &Y = *L;
    Y = Layout();
    Y.n = n;
    launches = 0;
    // sizes
    std::vector<JFrame> fr(n);
    for (int i = 0; i < n; ++i) {
        const JpegHeader &H = hd[i];
        JFrame &f = fr[i];
        std::memset(&f, 0, sizeof(f));
        f.w = H.w;
        f.h = H.h;
        f.ncomp = H.ncomp;
        f.bpm = H.bpm;
        f.mcux = H.mcux;
        f.mcuy = H.mcuy;
        f.hmax = H.hmax;
        f.vmax = H.vmax;
        f.ri = H.ri;
        f.nseg = H.nseg;
        f.seg_base = Y.n_seg;
        Y.n_seg += H.nseg;
        const size_t rl = len[i] - H.data_off;
        if (rl > (size_t)1 << 27) unsupported(i, "entropy-coded data larger than 128 MB");
        f.raw_len = (int)rl;
        f.raw_off = (long long)Y.raw_bytes;
        Y.raw_bytes += (rl + 16 + 15) & ~size_t(15);  // 16 bytes of slack: the bit reader loads 8 bytes at a time
        f.blk_base = Y.n_blocks;
        Y.n_blocks += H.blocks();
        f.sub_base = Y.n_sub;
        f.sub_bound = (int)(((long long)rl * 8 + kSubBits - 1) / kSubBits) + H.nseg;
        Y.n_sub += f.sub_bound;
        int k = 0;
        for (int c = 0; c < H.ncomp; ++c) {
            f.ch[c] = H.comp_h[c];
            f.cv[c] = H.comp_v[c];
            f.dc[c] = i * 8 + H.comp_dc[c];
            f.ac[c] = i * 8 + 4 + H.comp_ac[c];
            f.q[c] = H.comp_q[c];
            f.cw[c] = ceil_div(H.w * H.comp_h[c], H.hmax);
            f.chh[c] = ceil_div(H.h * H.comp_v[c], H.vmax);
            f.plane_pitch[c] = H.mcux * H.comp_h[c] * 8;
            f.plane_off[c] = (long long)Y.plane_bytes;
            Y.plane_bytes += a256((size_t)f.plane_pitch[c] * H.mcuy * H.comp_v[c] * 8);
            for (int by = 0; by < H.comp_v[c]; ++by)
                for (int bx = 0; bx < H.comp_h[c]; ++bx, ++k) {
                    f.lay_ci[k] = c;
                    f.lay_bx[k] = bx;
                    f.lay_by[k] = by;
                }
        }
    }
    Y.n_tab = 8 * n;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t r = o;
        o += a256(bytes);
        return r;
    };
    const size_t ns = (size_t)std::max(Y.n_seg, 1), nsub = (size_t)std::max(Y.n_sub, 1);
    Y.o_frames = take(sizeof(JFrame) * n);
    Y.o_tabs = take(sizeof(HuffTab) * Y.n_tab);
    Y.o_quant = take(sizeof(int32_t) * 64 * 4 * n);
    Y.o_seg_frame = take(sizeof(int) * ns);
    Y.o_seg_first = take(sizeof(long long) * ns);
    Y.o_seg_nblocks = take(sizeof(int) * ns);
    Y.o_raw = take(Y.raw_bytes);
    Y.upload = o;
    Y.o_ds = take(Y.raw_bytes);
    Y.o_seg_start = take(sizeof(int) * ns);
    Y.o_seg_bytes = take(sizeof(int) * ns);
    Y.o_seg_sub_base = take(sizeof(int) * ns);
    Y.o_seg_nsub = take(sizeof(int) * ns);
    Y.o_sub_seg = take(sizeof(int) * nsub);
    Y.o_st = take(sizeof(uint64_t) * nsub);
    Y.o_cnt = take(sizeof(int) * nsub);
    Y.o_ndc = take(sizeof(int) * nsub);
    Y.o_dcsum = take(sizeof(int) * 3 * nsub);
    Y.o_dcbase = take(sizeof(int) * 3 * nsub);
    Y.o_err = take(sizeof(int) * nsub);
    Y.o_blk_off = take(sizeof(long long) * nsub);
    Y.o_first_dc = take(sizeof(long long) * nsub);
    Y.o_status = take(sizeof(int) * (n + 1));
    Y.o_flag = Y.o_status + sizeof(int) * n;
    Y.o_coef = take(sizeof(int16_t) * 64 * (size_t)Y.n_blocks);
    Y.o_planes = take(Y.plane_bytes);
    Y.total = o;

    // staging: descriptors, tables, segment geometry and the entropy-coded bytes, in the workspace's layout
    // the previous call's copies and kernels on s are the only users of the old buffers (the flag words were read after a sync)
    if (Y.upload > h_stage.bytes() || Y.total > d_ws.bytes()) DFB_CUDA(cudaStreamSynchronize(s));
    h_stage.allocate(Y.upload);
    d_ws.allocate(Y.total);
    h_flag.allocate(sizeof(int) * std::max<size_t>(n + 1, 1024));
    uint8_t *S = h_stage;
    std::memcpy(S + Y.o_frames, fr.data(), sizeof(JFrame) * n);
    HuffTab *tabs = reinterpret_cast<HuffTab *>(S + Y.o_tabs);
    int32_t *quant = reinterpret_cast<int32_t *>(S + Y.o_quant);
    int *seg_frame = reinterpret_cast<int *>(S + Y.o_seg_frame), *seg_nblocks = reinterpret_cast<int *>(S + Y.o_seg_nblocks);
    long long *seg_first = reinterpret_cast<long long *>(S + Y.o_seg_first);
    for (int i = 0; i < n; ++i) {
        const JpegHeader &H = hd[i];
        for (int t = 0; t < 4; ++t) {
            if (H.dc[t].defined) build_table(H.dc[t], tabs[i * 8 + t]);
            if (H.ac[t].defined) build_table(H.ac[t], tabs[i * 8 + 4 + t]);
        }
        std::memcpy(quant + (size_t)i * 256, H.quant, sizeof(H.quant));
        const long long nmcu = (long long)H.mcux * H.mcuy, per = H.ri ? H.ri : nmcu;
        for (int g = 0; g < H.nseg; ++g) {
            seg_frame[fr[i].seg_base + g] = i;
            seg_first[fr[i].seg_base + g] = fr[i].blk_base + (long long)g * per * H.bpm;
            seg_nblocks[fr[i].seg_base + g] = (int)(std::min(per, nmcu - g * per) * H.bpm);
        }
        std::memcpy(S + Y.o_raw + fr[i].raw_off, jpeg[i] + H.data_off, fr[i].raw_len);
    }
    uint8_t *W = d_ws;
    DFB_CUDA(cudaMemcpyAsync(W, S, Y.upload, cudaMemcpyHostToDevice, s));
    DFB_CUDA(cudaMemsetAsync(W + Y.o_status, 0, sizeof(int) * (n + 1), s));
    DFB_CUDA(cudaMemsetAsync(W + Y.o_coef, 0, sizeof(int16_t) * 64 * (size_t)Y.n_blocks, s));

    EntropyArgs a{};
    a.ds = W + Y.o_ds;
    a.F = reinterpret_cast<const JFrame *>(W + Y.o_frames);
    a.tabs = reinterpret_cast<const HuffTab *>(W + Y.o_tabs);
    a.sub_seg = reinterpret_cast<int *>(W + Y.o_sub_seg);
    a.seg_sub_base = reinterpret_cast<int *>(W + Y.o_seg_sub_base);
    a.seg_nsub = reinterpret_cast<int *>(W + Y.o_seg_nsub);
    a.seg_start = reinterpret_cast<int *>(W + Y.o_seg_start);
    a.seg_bytes = reinterpret_cast<int *>(W + Y.o_seg_bytes);
    a.seg_frame = reinterpret_cast<int *>(W + Y.o_seg_frame);
    a.seg_nblocks = reinterpret_cast<int *>(W + Y.o_seg_nblocks);
    a.seg_first_block = reinterpret_cast<long long *>(W + Y.o_seg_first);
    a.st = reinterpret_cast<uint64_t *>(W + Y.o_st);
    a.cnt = reinterpret_cast<int *>(W + Y.o_cnt);
    a.ndc = reinterpret_cast<int *>(W + Y.o_ndc);
    a.dcsum = reinterpret_cast<int *>(W + Y.o_dcsum);
    a.dcbase = reinterpret_cast<int *>(W + Y.o_dcbase);
    a.err = reinterpret_cast<int *>(W + Y.o_err);
    a.blk_off = reinterpret_cast<long long *>(W + Y.o_blk_off);
    a.first_dc = reinterpret_cast<long long *>(W + Y.o_first_dc);
    a.coef = reinterpret_cast<int16_t *>(W + Y.o_coef);
    a.status = reinterpret_cast<int *>(W + Y.o_status);
    a.n_sub = Y.n_sub;
    a.n = n;
    int *d_flag = reinterpret_cast<int *>(W + Y.o_flag);

    k_destuff<<<n, kDT, 0, s>>>(W + Y.o_raw, W + Y.o_ds, a.F, reinterpret_cast<int *>(W + Y.o_seg_start),
                                reinterpret_cast<int *>(W + Y.o_seg_bytes), reinterpret_cast<int *>(W + Y.o_seg_sub_base),
                                reinterpret_cast<int *>(W + Y.o_seg_nsub), a.status);
    DFB_KERNEL_CHECK();
    const int gs = ceil_div(Y.n_sub, 128);
    k_init_states<<<ceil_div(Y.n_sub, 128), 128, 0, s>>>(a);
    DFB_KERNEL_CHECK();
    launches += 2;
    // rounds until no record changes; bounded by the longest segment's subsequence count (each round fixes at least the
    // first wrong record of every segment), which the total bounds
    sync_rounds = 0;
    for (int r = 0; r <= Y.n_sub; ++r) {
        DFB_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), s));
        k_sync_round<<<gs, 128, 0, s>>>(a, d_flag);
        DFB_KERNEL_CHECK();
        ++launches;
        ++sync_rounds;
        DFB_CUDA(cudaMemcpyAsync(h_flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
        DFB_CUDA(cudaStreamSynchronize(s));
        if (!h_flag[0]) break;
    }
    k_seg_scan<<<ceil_div(Y.n_seg * 32, 128), 128, 0, s>>>(a, Y.n_seg, 0);
    DFB_KERNEL_CHECK();
    k_decode_final<<<gs, 128, 0, s>>>(a);
    DFB_KERNEL_CHECK();
    k_seg_scan<<<ceil_div(Y.n_seg * 32, 128), 128, 0, s>>>(a, Y.n_seg, 1);
    DFB_KERNEL_CHECK();
    k_dc_fix<<<gs, 128, 0, s>>>(a);
    DFB_KERNEL_CHECK();
    launches += 4;
}

void JpegDecoder::check_status(int n, cudaStream_t s, int index_base) {
    DFB_CUDA(cudaMemcpyAsync(h_flag, d_ws + L->o_status, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
    for (int i = 0; i < n; ++i) {
        const int e = h_flag[i], f = index_base + i;
        if (e & kErrRst) corrupt(f, "wrong RST marker sequence in the entropy-coded data");
        if (e & kErrRstCount) corrupt(f, "the number of RST markers does not match the restart interval (truncated or corrupt data)");
        if (e & kErrCode) corrupt(f, "invalid Huffman code in the entropy-coded data");
        if (e & kErrShort) corrupt(f, "entropy-coded data ends before the last MCU");
        if (e & kErrNoEnd) corrupt(f, "entropy-coded data is not ended by a marker (truncated file)");
        if (e & kErrRange) corrupt(f, "dequantised DCT coefficient or IDCT output out of range (corrupt data)");
    }
}

void JpegDecoder::decode(const uint8_t *const *jpeg, const size_t *len, const JpegHeader *hd, int n, int channels, uint8_t *out,
                         size_t pitch, size_t frame_stride, cudaStream_t s, int index_base) {
    if (n <= 0) return;
    run_entropy(jpeg, len, hd, n, s);
    const Layout &Y = *L;
    const JFrame *F = reinterpret_cast<const JFrame *>(d_ws + Y.o_frames);
    if (Y.n_blocks > 0) {
        k_idct<<<(unsigned)((Y.n_blocks + 127) / 128), 128, 0, s>>>(reinterpret_cast<const int16_t *>(d_ws + Y.o_coef), F, n, Y.n_blocks,
                                                                   reinterpret_cast<const int32_t *>(d_ws + Y.o_quant), d_ws + Y.o_planes,
                                                                   reinterpret_cast<int *>(d_ws + Y.o_status));
        DFB_KERNEL_CHECK();
    }
    int mw = 0, mh = 0;
    for (int i = 0; i < n; ++i) {
        mw = std::max(mw, hd[i].w);
        mh = std::max(mh, hd[i].h);
    }
    k_color<<<dim3(ceil_div(ceil_div(mw, 2), 32), ceil_div(ceil_div(mh, 2), 8), n), dim3(32, 8), 0, s>>>(F, d_ws + Y.o_planes, channels, out,
                                                                                                          pitch, frame_stride);
    DFB_KERNEL_CHECK();
    launches += 2;
    check_status(n, s, index_base);
}

void JpegDecoder::coefficients(const uint8_t *jpeg, size_t len, const JpegHeader &hd, int16_t *out, cudaStream_t s) {
    run_entropy(&jpeg, &len, &hd, 1, s);
    check_status(1, s);
    DFB_CUDA(cudaMemcpyAsync(out, d_ws + L->o_coef, sizeof(int16_t) * 64 * (size_t)hd.blocks(), cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
}

}  // namespace dfb
