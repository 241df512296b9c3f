// png_encode.cu — imencode(".png", img) on the GPU, byte for byte: the last step of encodeFlowMapPng
// (src/common.cpp:66-71 of the reference).  Without IMWRITE_PNG_* parameters OpenCV's PNG encoder filters every row with SUB,
// and libpng compresses with zlib at level 1 (Z_BEST_SPEED) and strategy Z_RLE, in IDAT chunks of 8192 bytes.  Z_RLE only
// looks for matches at distance 1 and parses greedily, so the symbol stream splits into independent runs of equal bytes.
// Everything is integer arithmetic: the default and strict builds give the same bytes.
//
// A batch of n images of one size is encoded by one sequence of launches, blockIdx.y (or .z) spanning the images:
//   k_filter     scanlines: filter byte + RGB under SUB (NONE when w = 1), h * (1 + 3 w) bytes
//   k_tiles      per 4 KB tile: count of run starts and Adler-32 partials; zeroes the zlib stream buffer
//   k_scan       one CTA per image: exclusive scan of the tile counts -> run index bases, Adler-32 of the stream
//   k_runs       compacted run start positions
//   k_run_syms   per tile of runs: symbols the runs emit (png_deflate.cuh run_symbols, closed form)
//   k_scan       -> symbol index bases, symbol count, deflate block count (a flush every 16 383 symbols, then the final block)
//   k_sym_write  the symbols (uint16) and the byte position where each deflate block starts
//   k_blocks     one CTA per deflate block: histogram, then one thread runs zlib's tree construction and block choice
//   k_offsets    one warp per image: bit offset of every block (stored blocks byte-align), zlib header and Adler-32
//   k_emit       one CTA per deflate block: header bits, then every symbol's code at its prefix-summed bit offset
//   k_container  one warp per IDAT chunk: signature, IHDR, the chunk with its CRC-32 (slice CRCs combined), IEND
#include <algorithm>
#include <stdexcept>

#include "block_scan.cuh"
#include "common.cuh"
#include "png_deflate.cuh"
#include "png_encode.h"

namespace dfb {

namespace {

using namespace pngz;

constexpr int kTile = 4096;      // bytes (or runs) per tile
constexpr int kTileThreads = 256;
constexpr int kPer = kTile / kTileThreads;
constexpr int kIdat = 8192;      // libpng's compression buffer: bytes of zlib stream per IDAT chunk
constexpr size_t kWorkspaceBudget = size_t(512) << 20;  // images per launch sequence are capped by this much workspace

struct ImgInfo {
    uint32_t runs, nsym, nblocks, adler;
    uint32_t zlen, nchunks, error, pad;
    uint64_t file_len;
};

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Per-image workspace layout (all images of a batch have the same geometry)
struct Layout {
    uint32_t w, h, N, T, NB;
    size_t zcap, zwords, nchunks_max, file_cap;
    size_t o_run, o_sym, o_truns, o_tsyms, o_ts1, o_ts2, o_bpos, o_blocks, o_bstart, o_z, o_info, bytes;

    Layout(int w_, int h_) {
        w = w_, h = h_;
        N = (uint32_t)((size_t)h * (1 + 3 * (size_t)w));
        T = (N + kTile - 1) / kTile;
        NB = N / kBlockSyms + 2;
        // every block stored costs at most its bytes + 6 (3 bits, alignment, LEN / NLEN); + zlib header, Adler-32, slack
        zcap = (size_t)N + 8 * (size_t)NB + 16;
        zwords = zcap / 4 + 4;
        nchunks_max = (zcap + kIdat - 1) / kIdat;
        file_cap = 8 + 25 + zcap + 12 * nchunks_max + 12;
        size_t o = align256((size_t)N + 32);  // raw scanlines (16-byte loads may read past N)
        o_run = o, o = align256(o + 4 * ((size_t)N + 1));
        o_sym = o, o = align256(o + 2 * (size_t)N);
        o_truns = o, o = align256(o + 4 * (size_t)T);
        o_tsyms = o, o = align256(o + 4 * (size_t)T);
        o_ts1 = o, o = align256(o + 4 * (size_t)T);
        o_ts2 = o, o = align256(o + 4 * (size_t)T);
        o_bpos = o, o = align256(o + 4 * (size_t)NB);
        o_blocks = o, o = align256(o + sizeof(BlockInfo) * (size_t)NB);
        o_bstart = o, o = align256(o + 8 * (size_t)NB);
        o_z = o, o = align256(o + 4 * zwords);
        o_info = o, o = align256(o + sizeof(ImgInfo));
        bytes = o;
    }
    __device__ uint8_t *base(uint8_t *ws, int i) const { return ws + (size_t)i * bytes; }
    __device__ uint8_t *raw(uint8_t *ws, int i) const { return base(ws, i); }
    __device__ uint32_t *run(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_run); }
    __device__ uint16_t *sym(uint8_t *ws, int i) const { return (uint16_t *)(base(ws, i) + o_sym); }
    __device__ uint32_t *truns(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_truns); }
    __device__ uint32_t *tsyms(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_tsyms); }
    __device__ uint32_t *ts1(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_ts1); }
    __device__ uint32_t *ts2(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_ts2); }
    __device__ uint32_t *bpos(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_bpos); }
    __device__ BlockInfo *blocks(uint8_t *ws, int i) const { return (BlockInfo *)(base(ws, i) + o_blocks); }
    __device__ uint64_t *bstart(uint8_t *ws, int i) const { return (uint64_t *)(base(ws, i) + o_bstart); }
    __device__ uint32_t *z(uint8_t *ws, int i) const { return (uint32_t *)(base(ws, i) + o_z); }
    __device__ ImgInfo *info(uint8_t *ws, int i) const { return (ImgInfo *)(base(ws, i) + o_info); }
};

__device__ __forceinline__ void or_bits(uint32_t *zw, uint64_t off, uint32_t v, int len) {
    const uint64_t i = off >> 5;
    const int sh = (int)(off & 31);
    atomicOr(&zw[i], v << sh);
    if (sh + len > 32) atomicOr(&zw[i + 1], v >> (32 - sh));
}
__device__ __forceinline__ void or_byte(uint32_t *zw, uint64_t byte, uint32_t v) { atomicOr(&zw[byte >> 2], (v & 0xff) << (8 * (byte & 3))); }

// the 16 scanline bytes at p0 (16-aligned; the raw region has 32 bytes of slack past N), returns the byte before them
__device__ __forceinline__ uint8_t load16(const uint8_t *raw, size_t p0, uint32_t N, uint8_t *b) {
    if (p0 >= N) {
        *reinterpret_cast<uint4 *>(b) = make_uint4(0, 0, 0, 0);
        return 0;
    }
    *reinterpret_cast<uint4 *>(b) = *reinterpret_cast<const uint4 *>(raw + p0);
    return p0 ? raw[p0 - 1] : 0;
}

__global__ void k_filter(const uint8_t *src, size_t img_stride, size_t pitch, uint8_t *ws, Layout L) {
    const int img = blockIdx.z, y = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int rb = 1 + 3 * (int)L.w;
    if (i >= rb) return;
    const uint8_t *row = src + (size_t)img * img_stride + (size_t)y * pitch;
    uint8_t v;
    if (i == 0) {
        v = L.w == 1 ? 0 : 1;
    } else {  // libpng is told BGR, the file stores RGB; SUB subtracts the byte 3 to the left (0 left of the row)
        const int k = i - 1, p = k / 3, c = 2 - (k - 3 * p);
        v = (uint8_t)(row[3 * p + c] - (p ? row[3 * (p - 1) + c] : 0));
    }
    L.raw(ws, img)[(size_t)y * rb + i] = v;
}

__global__ void __launch_bounds__(kTileThreads) k_tiles(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, t = blockIdx.x;
    const uint8_t *raw = L.raw(ws, img);
    {  // zero this tile's share of the zlib stream buffer (the emitters OR into it)
        uint32_t *zw = L.z(ws, img);
        const size_t span = (L.zwords + L.T - 1) / L.T;
        for (size_t k = threadIdx.x; k < span; k += kTileThreads) {
            const size_t idx = (size_t)t * span + k;
            if (idx < L.zwords) zw[idx] = 0;
        }
    }
    const size_t p0 = (size_t)t * kTile + threadIdx.x * kPer;
    uint8_t b[kPer];
    uint8_t prev = load16(raw, p0, L.N, b);
    uint32_t runs = 0, s1 = 0, s2 = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
        if (p0 + j < L.N) {
            runs += (p0 + j == 0 || b[j] != prev);
            s1 += b[j];
            s2 += (kPer - j) * b[j];
        }
        prev = b[j];
    }
    // Adler-32 partials: s1 = sum of bytes, s2 = sum of (tile end - p) * byte
    const uint64_t s2t = s2 + (uint64_t)(kTileThreads - 1 - threadIdx.x) * kPer * s1;
    __shared__ uint32_t sm32[kTileThreads / 32];
    __shared__ uint64_t sm64[kTileThreads / 32];
    const uint32_t truns = block_sum<kTileThreads>(runs, sm32);
    const uint32_t ts1 = block_sum<kTileThreads>(s1, sm32);
    const uint64_t ts2 = block_sum<kTileThreads>(s2t, sm64);
    if (threadIdx.x == 0) {
        L.truns(ws, img)[t] = truns;
        L.ts1(ws, img)[t] = ts1 % kAdlerMod;
        L.ts2(ws, img)[t] = (uint32_t)(ts2 % kAdlerMod);
    }
}

// which = 0: run counts of the byte tiles (+ Adler-32); which = 1: symbol counts of the run tiles
__global__ void __launch_bounds__(1024) k_scan(uint8_t *ws, Layout L, int which) {
    const int img = blockIdx.x;
    uint32_t *a = which == 0 ? L.truns(ws, img) : L.tsyms(ws, img);
    const uint32_t T = L.T, per = (T + 1023) / 1024, lo = min(T, threadIdx.x * per), hi = min(T, lo + per);
    __shared__ uint32_t sm32[32];
    __shared__ uint64_t sm64[32];
    uint32_t sum = 0;
    for (uint32_t i = lo; i < hi; ++i) sum += a[i];
    uint32_t total;
    uint32_t run = block_scan<1024>(sum, total, sm32);
    for (uint32_t i = lo; i < hi; ++i) {
        const uint32_t v = a[i];
        a[i] = run;
        run += v;
    }
    ImgInfo *info = L.info(ws, img);
    if (which == 0) {
        // Adler-32: a = 1 + sum of bytes, b = N + sum of (N - p) * byte, modulo 65521
        const uint32_t *ts1 = L.ts1(ws, img), *ts2 = L.ts2(ws, img);
        uint64_t s1 = 0, s2 = 0;
        for (uint32_t i = lo; i < hi; ++i) {
            const int64_t d = (int64_t)L.N - (int64_t)(i + 1) * kTile;  // N - tile end (negative for the last tile)
            const uint64_t dm = (uint64_t)(((d % (int64_t)kAdlerMod) + kAdlerMod) % kAdlerMod);
            s1 += ts1[i];
            s2 += ts2[i] + dm * ts1[i] % kAdlerMod;
        }
        s1 = block_sum<1024>(s1 % kAdlerMod, sm64);
        s2 = block_sum<1024>(s2 % kAdlerMod, sm64);
        if (threadIdx.x == 0) {
            const uint32_t A = (uint32_t)((1 + s1) % kAdlerMod), B = (uint32_t)((L.N % kAdlerMod + s2) % kAdlerMod);
            info->adler = B << 16 | A;
            info->runs = total;
            L.run(ws, img)[total] = L.N;  // sentinel: the end of the last run
        }
    } else if (threadIdx.x == 0) {
        info->nsym = total;
        info->nblocks = total / kBlockSyms + 1;
        if (total % kBlockSyms == 0) L.bpos(ws, img)[total / kBlockSyms] = L.N;  // the empty final block
    }
}

__global__ void __launch_bounds__(kTileThreads) k_runs(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, t = blockIdx.x;
    const uint8_t *raw = L.raw(ws, img);
    const size_t p0 = (size_t)t * kTile + threadIdx.x * kPer;
    uint8_t b[kPer];
    uint8_t prev = load16(raw, p0, L.N, b);
    uint32_t flags = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
        if (p0 + j < L.N && (p0 + j == 0 || b[j] != prev)) flags |= 1u << j;
        prev = b[j];
    }
    __shared__ uint32_t sm[kTileThreads / 32];
    uint32_t total;
    uint32_t o = L.truns(ws, img)[t] + block_scan<kTileThreads>((uint32_t)__popc(flags), total, sm);
    uint32_t *run = L.run(ws, img);
    while (flags) {
        const int j = __ffs(flags) - 1;
        flags &= flags - 1;
        run[o++] = (uint32_t)(p0 + j);
    }
}

__global__ void __launch_bounds__(kTileThreads) k_run_syms(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, t = blockIdx.x;
    const uint32_t R = L.info(ws, img)->runs, *run = L.run(ws, img);
    const uint32_t r0 = t * kTile + threadIdx.x * kPer;
    uint32_t c = 0;
    for (int j = 0; j < kPer; ++j)
        if (r0 + j < R) c += run_symbols(run[r0 + j + 1] - run[r0 + j]);
    __shared__ uint32_t sm[kTileThreads / 32];
    c = block_sum<kTileThreads>(c, sm);
    if (threadIdx.x == 0) L.tsyms(ws, img)[t] = c;
}

__global__ void __launch_bounds__(kTileThreads) k_sym_write(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, t = blockIdx.x;
    const uint32_t R = L.info(ws, img)->runs, *run = L.run(ws, img);
    const uint32_t r0 = t * kTile + threadIdx.x * kPer;
    if ((uint32_t)t * kTile >= R) return;  // whole CTA past the last run
    uint32_t c = 0;
    for (int j = 0; j < kPer; ++j)
        if (r0 + j < R) c += run_symbols(run[r0 + j + 1] - run[r0 + j]);
    __shared__ uint32_t sm[kTileThreads / 32];
    uint32_t total;
    uint32_t i = L.tsyms(ws, img)[t] + block_scan<kTileThreads>(c, total, sm);
    const uint8_t *raw = L.raw(ws, img);
    uint16_t *sym = L.sym(ws, img);
    uint32_t *bpos = L.bpos(ws, img);
    auto put = [&](uint16_t v, uint32_t pos) {
        if (i % kBlockSyms == 0) bpos[i / kBlockSyms] = pos;
        sym[i++] = v;
    };
    for (int j = 0; j < kPer && r0 + j < R; ++j) {
        const uint32_t s = run[r0 + j], n = run[r0 + j + 1] - s, r = n - 1;
        const uint16_t lit = raw[s];
        put(lit, s);
        uint32_t k = 0;
        for (uint32_t m = run_matches(n); m; --m) {
            const uint32_t len = min(r - k, 258u);
            put((uint16_t)(256 + len - 3), s + 1 + k);
            k += len;
        }
        for (; k < r; ++k) put(lit, s + 1 + k);
    }
}

constexpr int kBlockThreads = 128;

__global__ void __launch_bounds__(kBlockThreads) k_blocks(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, b = blockIdx.x;
    const ImgInfo *info = L.info(ws, img);
    const uint32_t nblocks = info->nblocks, S = info->nsym;
    if ((uint32_t)b >= nblocks) return;
    __shared__ Trees tw;
    __shared__ BlockInfo bi;
    __shared__ uint32_t lfreq[kLCodes], dfreq;
    for (int k = threadIdx.x; k < (int)(sizeof(Trees) / 4); k += kBlockThreads) reinterpret_cast<uint32_t *>(&tw)[k] = 0;
    for (int k = threadIdx.x; k < (int)(sizeof(BlockInfo) / 4); k += kBlockThreads) reinterpret_cast<uint32_t *>(&bi)[k] = 0;
    for (int k = threadIdx.x; k < kLCodes; k += kBlockThreads) lfreq[k] = 0;
    if (threadIdx.x == 0) dfreq = 0;
    __syncthreads();
    const uint32_t i0 = (uint32_t)b * kBlockSyms, i1 = min(S, i0 + kBlockSyms);
    const uint16_t *sym = L.sym(ws, img);
    uint32_t matches = 0;
    for (uint32_t i = i0 + threadIdx.x; i < i1; i += kBlockThreads) {
        const uint16_t v = sym[i];
        if (v < 256) {
            atomicAdd(&lfreq[v], 1u);
        } else {
            atomicAdd(&lfreq[257 + length_code(v - 256)], 1u);
            ++matches;
        }
    }
    if (matches) atomicAdd(&dfreq, matches);
    __syncthreads();
    for (int k = threadIdx.x; k < kLCodes; k += kBlockThreads) tw.ltree[k].fc = (uint16_t)(k == kEndBlock ? 1 : lfreq[k]);
    if (threadIdx.x == 0) {
        tw.dtree[0].fc = (uint16_t)dfreq;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t *bpos = L.bpos(ws, img);
        const uint32_t pos = bpos[b], end = (uint32_t)b + 1 < nblocks ? bpos[b + 1] : L.N;
        flush_block(tw, end - pos, (uint32_t)b + 1 == nblocks, bi);
        bi.pos = pos;
        bi.first_sym = i0;
        bi.nsym = i1 - i0;
    }
    __syncthreads();
    uint32_t *dst = reinterpret_cast<uint32_t *>(L.blocks(ws, img) + b);
    for (int k = threadIdx.x; k < (int)(sizeof(BlockInfo) / 4); k += kBlockThreads) dst[k] = reinterpret_cast<const uint32_t *>(&bi)[k];
}

__global__ void __launch_bounds__(32) k_offsets(uint8_t *ws, Layout L) {
    const int img = blockIdx.x, lane = threadIdx.x;
    ImgInfo *info = L.info(ws, img);
    const uint32_t nb = info->nblocks;
    const BlockInfo *blk = L.blocks(ws, img);
    uint64_t *bstart = L.bstart(ws, img);
    uint64_t off = 16;  // after the 2-byte zlib header
    for (uint32_t base = 0; base < nb; base += 32) {
        uint32_t type = 0, bits = 0, len = 0;
        if (base + lane < nb) {
            type = blk[base + lane].type;
            bits = blk[base + lane].bits;
            len = blk[base + lane].len;
        }
        const uint32_t cnt = min(32u, nb - base);
        for (uint32_t k = 0; k < cnt; ++k) {
            const uint32_t tk = __shfl_sync(0xffffffffu, type, k), bk = __shfl_sync(0xffffffffu, bits, k), lk = __shfl_sync(0xffffffffu, len, k);
            if (lane == (int)k) bstart[base + k] = off;
            off = tk == kStored ? ((off + 3 + 7) & ~uint64_t(7)) + 32 + 8 * (uint64_t)lk : off + bk;
        }
    }
    if (lane != 0) return;
    const uint64_t zb = (off + 7) / 8, Z = zb + 4;
    if (Z > L.zcap) {  // cannot happen (see Layout); fail the image rather than write past the buffer
        info->error = 1;
        return;
    }
    info->error = 0;
    uint32_t *zw = L.z(ws, img);
    uint32_t cinfo = 7;  // libpng declares the smallest window that covers the data
    while (cinfo > 0 && (1ull << (cinfo + 7)) >= L.N) cinfo--;
    const uint32_t cmf = cinfo << 4 | 8;
    or_byte(zw, 0, cmf);
    or_byte(zw, 1, 31 - (cmf * 256) % 31);
    const uint32_t ad = info->adler;
    for (int k = 0; k < 4; ++k) or_byte(zw, zb + k, ad >> (24 - 8 * k));
    info->zlen = (uint32_t)Z;
    info->nchunks = (uint32_t)((Z + kIdat - 1) / kIdat);
    info->file_len = 8 + 25 + Z + 12 * (uint64_t)info->nchunks + 12;
}

constexpr int kEmitThreads = 256;

__global__ void __launch_bounds__(kEmitThreads) k_emit(uint8_t *ws, Layout L) {
    const int img = blockIdx.y, b = blockIdx.x;
    const ImgInfo *info = L.info(ws, img);
    if ((uint32_t)b >= info->nblocks || info->error) return;
    const BlockInfo &B = L.blocks(ws, img)[b];
    const uint64_t start = L.bstart(ws, img)[b];
    uint32_t *zw = L.z(ws, img);
    const uint32_t type = B.type;
    if (type == kStored) {
        const uint32_t len = B.len, pos = B.pos;
        const uint64_t q = (start + 3 + 7) >> 3;
        if (threadIdx.x == 0) {
            or_bits(zw, start, B.last, 3);
            or_byte(zw, q, len);
            or_byte(zw, q + 1, len >> 8);
            or_byte(zw, q + 2, ~len);
            or_byte(zw, q + 3, ~len >> 8);
        }
        const uint8_t *raw = L.raw(ws, img) + pos;
        for (uint32_t k = threadIdx.x; k < len; k += kEmitThreads) or_byte(zw, q + 4 + k, raw[k]);
        return;
    }
    __shared__ uint32_t lit[kLCodes];
    __shared__ uint32_t sm[kEmitThreads / 32];
    for (int k = threadIdx.x; k < kLCodes; k += kEmitThreads) lit[k] = B.lit[k];
    const uint32_t dist = B.dist, hdr_bits = B.hdr_bits;
    for (uint32_t k = threadIdx.x; 32 * k < hdr_bits; k += kEmitThreads) or_bits(zw, start + 32 * k, B.hdr[k], min(32u, hdr_bits - 32 * k));
    __syncthreads();
    const uint32_t nsym = B.nsym, items = nsym + 1;  // + end of block
    const uint32_t per = (items + kEmitThreads - 1) / kEmitThreads, lo = min(items, threadIdx.x * per), hi = min(items, lo + per);
    const uint16_t *sym = L.sym(ws, img) + B.first_sym;
    uint32_t mine = 0;
    for (uint32_t k = lo; k < hi; ++k) {
        uint32_t v;
        mine += symbol_bits(k < nsym ? sym[k] : kSymEob, lit, dist, v);
    }
    uint32_t total;
    const uint64_t o = start + hdr_bits + block_scan<kEmitThreads>(mine, total, sm);
    // words entirely inside this thread's bits are stored; the partial first and last words are ORed
    uint64_t wi = o >> 5, acc = 0;
    int nbit = (int)(o & 31);
    bool shared = nbit != 0;
    for (uint32_t k = lo; k < hi; ++k) {
        uint32_t v;
        const int len = symbol_bits(k < nsym ? sym[k] : kSymEob, lit, dist, v);
        acc |= (uint64_t)v << nbit;
        nbit += len;
        if (nbit >= 32) {
            if (shared) atomicOr(&zw[wi], (uint32_t)acc);
            else zw[wi] = (uint32_t)acc;
            shared = false;
            acc >>= 32;
            nbit -= 32;
            ++wi;
        }
    }
    if (acc) atomicOr(&zw[wi], (uint32_t)acc);
}

__device__ __forceinline__ void put_be32(uint8_t *p, uint32_t v) {
    p[0] = v >> 24;
    p[1] = v >> 16;
    p[2] = v >> 8;
    p[3] = v;
}

__device__ uint32_t crc_bytes(uint32_t reg, const uint8_t *p, uint32_t n, const uint32_t *tab) {
    for (uint32_t k = 0; k < n; ++k) reg = tab[(reg ^ p[k]) & 0xff] ^ (reg >> 8);
    return reg;
}

__global__ void __launch_bounds__(32) k_container(uint8_t *ws, Layout L, uint8_t *files, size_t file_cap, uint64_t *lens) {
    const int img = blockIdx.y, c = blockIdx.x, lane = threadIdx.x;
    const ImgInfo *info = L.info(ws, img);
    if (info->error) {
        if (c == 0 && lane == 0) lens[img] = 0;
        return;
    }
    const uint32_t nchunks = info->nchunks, Z = info->zlen;
    if ((uint32_t)c >= nchunks) return;
    __shared__ uint32_t tab[256];
    for (int k = lane; k < 256; k += 32) {
        uint32_t v = k;
        for (int j = 0; j < 8; ++j) v = v & 1 ? (v >> 1) ^ kCrcPoly : v >> 1;
        tab[k] = v;
    }
    __syncwarp();
    const uint8_t *zb = reinterpret_cast<const uint8_t *>(L.z(ws, img));
    uint8_t *file = files + (size_t)img * file_cap;
    if (c == 0 && lane == 0) {
        const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
        for (int k = 0; k < 8; ++k) file[k] = sig[k];
        uint8_t *ih = file + 8;  // IHDR: width, height, bit depth 8, colour type 2 (RGB), deflate, adaptive filtering, no interlace
        put_be32(ih, 13);
        ih[4] = 'I', ih[5] = 'H', ih[6] = 'D', ih[7] = 'R';
        put_be32(ih + 8, L.w);
        put_be32(ih + 12, L.h);
        ih[16] = 8, ih[17] = 2, ih[18] = 0, ih[19] = 0, ih[20] = 0;
        put_be32(ih + 21, ~crc_bytes(0xffffffffu, ih + 4, 17, tab));
        lens[img] = info->file_len;
    }
    const uint32_t p0 = (uint32_t)c * kIdat, n = min((uint32_t)kIdat, Z - p0);
    uint8_t *out = file + 33 + (size_t)c * (kIdat + 12);
    for (uint32_t k = lane; k < n; k += 32) out[8 + k] = zb[p0 + k];
    // CRC-32 of "IDAT" + data: each lane runs the register from 0 over its slice, shifted past the bytes after it
    constexpr uint32_t kSlice = kIdat / 32;
    const uint32_t lo = min(n, lane * kSlice), hi = min(n, lo + kSlice);
    uint32_t part = 0;
    if (lo < hi) part = multmodp(x8nmodp(n - hi), crc_bytes(0, zb + p0 + lo, hi - lo, tab));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part ^= __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) {
        put_be32(out, n);
        out[4] = 'I', out[5] = 'D', out[6] = 'A', out[7] = 'T';
        const uint32_t reg = crc_bytes(0xffffffffu, out + 4, 4, tab);
        put_be32(out + 8 + n, ~(multmodp(x8nmodp(n), reg) ^ part));
        if ((uint32_t)c + 1 == nchunks) {
            uint8_t *ie = out + 12 + n;
            put_be32(ie, 0);
            ie[4] = 'I', ie[5] = 'E', ie[6] = 'N', ie[7] = 'D';
            put_be32(ie + 8, 0xAE426082u);
        }
    }
}

}  // namespace

size_t png_max_bytes(int w, int h) {
    if (w <= 0 || h <= 0) return 0;
    return Layout(w, h).file_cap;
}

int PngEncoder::encode(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, int slot, cudaStream_t s) {
    if (n <= 0) return 0;
    if ((size_t)h * (1 + 3 * (size_t)w) >= (size_t(1) << 31)) throw std::runtime_error("png: image too large");
    const Layout L(w, h);
    files_.prepare(slot, n, L.file_cap);
    const int E = (int)std::max<size_t>(1, std::min<size_t>((size_t)n, kWorkspaceBudget / L.bytes));
    ws_.grow((size_t)E * L.bytes);
    int launches = 0;
    for (int i0 = 0; i0 < n; i0 += E)
        launches += encode_part(std::min(E, n - i0), src + (size_t)i0 * img_stride, img_stride, bgr_pitch, w, h, files_.file(slot, i0),
                                files_.lens(slot) + i0, s);
    files_.read_lens(slot, n, s);
    return launches;
}

int PngEncoder::encode_part(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, uint8_t *files, uint64_t *lens,
                            cudaStream_t s) {
    const Layout L(w, h);
    const int rb = 1 + 3 * w;
    k_filter<<<dim3(ceil_div(rb, 256), h, n), 256, 0, s>>>(src, img_stride, bgr_pitch, ws_, L);
    DFB_KERNEL_CHECK();
    k_tiles<<<dim3(L.T, n), kTileThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_scan<<<n, 1024, 0, s>>>(ws_, L, 0);
    DFB_KERNEL_CHECK();
    k_runs<<<dim3(L.T, n), kTileThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_run_syms<<<dim3(L.T, n), kTileThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_scan<<<n, 1024, 0, s>>>(ws_, L, 1);
    DFB_KERNEL_CHECK();
    k_sym_write<<<dim3(L.T, n), kTileThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_blocks<<<dim3(L.NB, n), kBlockThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_offsets<<<n, 32, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_emit<<<dim3(L.NB, n), kEmitThreads, 0, s>>>(ws_, L);
    DFB_KERNEL_CHECK();
    k_container<<<dim3((unsigned)L.nchunks_max, n), 32, 0, s>>>(ws_, L, files, L.file_cap, lens);
    DFB_KERNEL_CHECK();
    return 11;
}

}  // namespace dfb
