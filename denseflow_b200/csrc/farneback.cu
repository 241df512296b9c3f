// farneback.cu — the Farneback path on sm_90a: what cv::cuda::FarnebackOpticalFlow::calc executes with
// the argument-less create() defaults the reference uses (/root/reference/src/denseflow_gpu.cpp:301,329;
// arithmetic per SURVEY.md Appendix B: numLevels 5, pyrScale .5, winSize 13, numIters 10, polyN 5,
// polySigma 1.1, flags 0 = box filter).
//
// Per level (coarse -> fine): Gaussian blur of the FULL-resolution frame + bilinear resize to the level
// (B.2), polynomial expansion (B.3), then 10 x [13x13 box mean of the five M planes -> per-pixel 2x2
// solve -> rebuild M] (B.4, B.5).  Two create() options change that (B.7): "gaussian_window"
// (OPTFLOW_FARNEBACK_GAUSSIAN) averages M over a 13x13 Gaussian window instead of the box, and "fast_pyramids" builds the
// level images by a chain of pyrDown from the unblurred frame instead of blur + resize.  All planes are fp32 with 128-byte-aligned rows; the five planes of
// R / M are stored as five separate planes of one pitch (the reference stacks them in a 5H x W matrix).
// These kernels are HBM-bound 2-D stencils: separable passes staged through shared-memory tiles,
// float4 on the interior, index-clamp / reflect-101 border rules applied on image coordinates.
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "engine.h"
#include "tma.cuh"
#include "tvl1.cuh"

namespace dfb {

namespace {

constexpr int kMaxLevels = 8;
constexpr int kMaxHalf = 40;  // largest Gaussian half-width: level k = 5 has sigma 15.5 -> smoothSize 79 -> half 39

struct FarnConsts {
    float g[8], xg[8], xxg[8];  // polyN <= 7
    float ig11, ig03, ig33, ig55;
};

struct Plane5 {
    float *p[5];
    int w, h, pitch;
};

__host__ __device__ inline int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}

// ---- B.2 Gaussian blur, separable, BORDER_REFLECT_101; vertical pass first (upstream order) -------
// One CTA computes a 32 x 32 output tile: stage (32 + 2*half) rows x 32 cols vertically filtered... the
// vertical pass needs rows y-half..y+half of the source; the horizontal pass needs the vertically
// filtered values at x-half..x+half.  So: vertical-filter a (32 + 2*half)-wide strip of 32 rows into
// shared memory, then filter horizontally out of shared memory.
struct GaussKernel {
    float k[kMaxHalf + 1];
    int half;
};

constexpr int GT = 32;  // tile edge

// Frame preparation is batched like the pairs: every stage is launched once for all the new frames of a batch (blockIdx.z =
// frame).  At these sizes each stage is launch-latency-bound (~18 small launches per frame), so a 17-frame batch went from ~300
// launches to 18.
constexpr int kMaxPrep = 16;
struct PrepBatch {
    const uint8_t *src[kMaxPrep];
    float *frame[kMaxPrep], *vn[kMaxPrep], *img[kMaxPrep];
    float *r[kMaxPrep];  // first R plane of the current level in the frame's slot
};

__global__ void k_farn_u8_to_f32(const __grid_constant__ PrepBatch pb, size_t src_pitch, int w, int h, int pitch) {
    const int x0 = 4 * (blockIdx.x * 32 + threadIdx.x), y = blockIdx.y * 8 + threadIdx.y;
    if (y >= h || x0 >= w) return;
    const uint8_t *row = pb.src[blockIdx.z] + (size_t)y * src_pitch;
    float4 v;
    v.x = row[x0];
    v.y = x0 + 1 < w ? row[x0 + 1] : 0.f;
    v.z = x0 + 2 < w ? row[x0 + 2] : 0.f;
    v.w = x0 + 3 < w ? row[x0 + 3] : 0.f;
    *reinterpret_cast<float4 *>(pb.frame[blockIdx.z] + (size_t)y * pitch + x0) = v;  // pitch % 32 == 0: in-bounds
}

__global__ void __launch_bounds__(256) k_gauss_blur(const __grid_constant__ PrepBatch pb, int fw, int fh, int fpitch, const GaussKernel gk) {
    const Plane src{pb.frame[blockIdx.z], fw, fh, fpitch}, dst{pb.img[blockIdx.z], fw, fh, fpitch};
    extern __shared__ float smem[];  // [GT][GT + 2*half]
    const int half = gk.half;
    const int sw = GT + 2 * half;
    const int x0 = blockIdx.x * GT, y0 = blockIdx.y * GT;
    // vertical pass into shared memory
    for (int i = threadIdx.x; i < GT * sw; i += blockDim.x) {
        const int ty = i / sw, tx = i - ty * sw;
        const int y = min(y0 + ty, src.h - 1);
        const int x = reflect101(x0 + tx - half, src.w);
        float acc = src.p[(size_t)y * src.pitch + x] * gk.k[0];
        for (int j = 1; j <= half; ++j)
            acc = acc + (src.p[(size_t)reflect101(y - j, src.h) * src.pitch + x] + src.p[(size_t)reflect101(y + j, src.h) * src.pitch + x]) * gk.k[j];
        smem[i] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < GT * GT; i += blockDim.x) {
        const int ty = i / GT, tx = i - ty * GT;
        const int x = x0 + tx, y = y0 + ty;
        if (x >= dst.w || y >= dst.h) continue;
        const float *row = smem + ty * sw + tx + half;
        float acc = row[0] * gk.k[0];
        for (int j = 1; j <= half; ++j) acc = acc + (row[-j] + row[j]) * gk.k[j];
        dst.p[(size_t)y * dst.pitch + x] = acc;
    }
}

// ---- B.2 fused for levels with scale < 1: blur + resize, evaluated only where the resize looks -----------------
// The reference blurs the WHOLE full-resolution frame for every level and then samples it with a bilinear resize that
// reads just two rows / two columns per level pixel.  These two kernels compute exactly those samples — the vertical
// pass only on the 2 * H_level rows the resize touches, the horizontal pass only at the 2 x 2 taps of each level pixel —
// with the same operation order per value (vertical first; centre tap, then symmetric pairs), so the level image is
// bit-identical to blur-then-resize while the work drops from ~70 to ~24 taps per full-resolution pixel and level set.
__global__ void __launch_bounds__(256) k_gauss_vert_rows(const __grid_constant__ PrepBatch pb, int fw, int fh, int fpitch, int lh, float rfy,
                                                         const GaussKernel gk) {
    const Plane src{pb.frame[blockIdx.z], fw, fh, fpitch}, vn{pb.vn[blockIdx.z], fw, 2 * lh, fpitch};  // vn: 2 * H_level rows
    const int x = blockIdx.x * 256 + threadIdx.x;
    const int ri = blockIdx.y;  // row pair index: level row ri >> 1, tap ri & 1
    if (x >= src.w) return;
    const float sy = (ri >> 1) * rfy;
    const int y1 = __float2int_rd(sy);
    const int y = (ri & 1) ? min(y1 + 1, src.h - 1) : min(y1, src.h - 1);
    float acc = src.p[(size_t)y * src.pitch + x] * gk.k[0];
    for (int j = 1; j <= gk.half; ++j)
        acc = acc + (src.p[(size_t)reflect101(y - j, src.h) * src.pitch + x] + src.p[(size_t)reflect101(y + j, src.h) * src.pitch + x]) * gk.k[j];
    vn.p[(size_t)ri * vn.pitch + x] = acc;
}

__global__ void __launch_bounds__(256) k_gauss_horz_resize(const __grid_constant__ PrepBatch pb, int src_w, int src_h, int fpitch, int lw, int lh,
                                                           int lpitch, float rfx, float rfy, const GaussKernel gk) {
    const Plane vn{pb.vn[blockIdx.z], src_w, 2 * lh, fpitch}, dst{pb.img[blockIdx.z], lw, lh, lpitch};
    const int dx = blockIdx.x * 32 + threadIdx.x, dy = blockIdx.y * 8 + threadIdx.y;
    if (dx >= dst.w || dy >= dst.h) return;
    const float sx = dx * rfx, sy = dy * rfy;
    const int x1 = __float2int_rd(sx), y1 = __float2int_rd(sy);
    const int x2 = x1 + 1, y2 = y1 + 1;
    const int xc[2] = {min(x1, src_w - 1), min(x2, src_w - 1)};
    (void)src_h;
    float b[2][2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const float *row = vn.p + (size_t)(2 * dy + r) * vn.pitch;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            float acc = row[xc[c]] * gk.k[0];
            for (int j = 1; j <= gk.half; ++j) acc = acc + (row[reflect101(xc[c] - j, src_w)] + row[reflect101(xc[c] + j, src_w)]) * gk.k[j];
            b[r][c] = acc;
        }
    }
    float out = 0.f;  // same accumulation order as k_resize_linear
    out = out + b[0][0] * ((x2 - sx) * (y2 - sy));
    out = out + b[0][1] * ((sx - x1) * (y2 - sy));
    out = out + b[1][0] * ((x2 - sx) * (sy - y1));
    out = out + b[1][1] * ((sx - x1) * (sy - y1));
    dst.p[(size_t)dy * dst.pitch + dx] = out;
}

// ---- B.7 fastPyramids: level k = pyrDown(level k - 1), batched like the preparation stages (blockIdx.z = frame) --------------
// cv::cuda::pyrDown, BORDER_REFLECT_101: output (x, y) is the 5-tap [1 4 6 4 1] / 16 filter at source column / row 2x / 2y,
// the vertical pass first, each pass summed left to right in fp32.  The 25 taps of a pixel come through L1; the levels it
// runs on are a quarter of the frame and smaller.
struct PyrBatch {
    const float *src[kMaxPrep];
    float *dst[kMaxPrep];
};

__global__ void __launch_bounds__(256) k_pyr_down(const __grid_constant__ PyrBatch pb, int sw, int sh, int spitch, int dw, int dh, int dpitch) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const float *src = pb.src[blockIdx.z];
    const float k[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    size_t rows[5];
#pragma unroll
    for (int d = 0; d < 5; ++d) rows[d] = (size_t)reflect101(2 * y + d - 2, sh) * spitch;
    float out = 0.f;
#pragma unroll
    for (int e = 0; e < 5; ++e) {
        const int c = reflect101(2 * x + e - 2, sw);
        float v = src[rows[0] + c] * k[0];
#pragma unroll
        for (int d = 1; d < 5; ++d) v = v + src[rows[d] + c] * k[d];
        out = e == 0 ? v * k[0] : out + v * k[e];
    }
    pb.dst[blockIdx.z][(size_t)y * dpitch + x] = out;
}

// ---- B.3 polynomial expansion (polyN = 5): vertical pass (t0,t1,t2) then horizontal, index-clamped ----
constexpr int PT = 32;

template <int N>
__global__ void __launch_bounds__(256) k_poly_exp(const __grid_constant__ PrepBatch pb, int lw, int lh, int lpitch, size_t plane_elems, const FarnConsts c) {
    const Plane src{pb.img[blockIdx.z], lw, lh, lpitch};
    float *const rb = pb.r[blockIdx.z];
    const Plane5 R{{rb, rb + plane_elems, rb + 2 * plane_elems, rb + 3 * plane_elems, rb + 4 * plane_elems}, lw, lh, lpitch};
    __shared__ float t0[PT][PT + 2 * N], t1[PT][PT + 2 * N], t2[PT][PT + 2 * N];
    constexpr int sw = PT + 2 * N;
    const int x0 = blockIdx.x * PT, y0 = blockIdx.y * PT;
    for (int i = threadIdx.x; i < PT * sw; i += blockDim.x) {
        const int ty = i / sw, tx = i - ty * sw;
        const int y = min(y0 + ty, src.h - 1);
        const int x = max(0, min(x0 + tx - N, src.w - 1));
        float a0 = src.p[(size_t)y * src.pitch + x] * c.g[0], a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 1; k <= N; ++k) {
            const float s0 = src.p[(size_t)max(y - k, 0) * src.pitch + x];
            const float s1 = src.p[(size_t)min(y + k, src.h - 1) * src.pitch + x];
            a0 = a0 + c.g[k] * (s0 + s1);
            a1 = a1 + c.xg[k] * (s1 - s0);
            a2 = a2 + c.xxg[k] * (s0 + s1);
        }
        t0[ty][tx] = a0;
        t1[ty][tx] = a1;
        t2[ty][tx] = a2;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < PT * PT; i += blockDim.x) {
        const int ty = i / PT, tx = i - ty * PT;
        const int x = x0 + tx, y = y0 + ty;
        if (x >= src.w || y >= src.h) continue;
        const float *r0 = &t0[ty][tx + N], *r1 = &t1[ty][tx + N], *r2 = &t2[ty][tx + N];
        float b1 = c.g[0] * r0[0], b3 = c.g[0] * r1[0], b5 = c.g[0] * r2[0], b2 = 0.f, b4 = 0.f, b6 = 0.f;
#pragma unroll
        for (int k = 1; k <= N; ++k) {
            float s = r0[k] + r0[-k];
            b1 = b1 + s * c.g[k];
            b4 = b4 + s * c.xxg[k];
            b2 = b2 + (r0[k] - r0[-k]) * c.xg[k];
            s = r1[k] + r1[-k];
            b3 = b3 + s * c.g[k];
            b6 = b6 + (r1[k] - r1[-k]) * c.xg[k];
            s = r2[k] + r2[-k];
            b5 = b5 + s * c.g[k];
        }
        const size_t o = (size_t)y * R.pitch + x;
        R.p[0][o] = b3 * c.ig11;
        R.p[1][o] = b2 * c.ig11;
        R.p[2][o] = b1 * c.ig03 + b5 * c.ig33;
        R.p[3][o] = b1 * c.ig03 + b4 * c.ig33;
        R.p[4][o] = b6 * c.ig55;
    }
}

__constant__ float c_border[6] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f, 1.f};
// B.7 Gaussian window: getGaussianKernel(13, 6 * 0.3f, CV_32F), centre and right half (set by the engine's constructor)
__constant__ float c_gauss_win[7];

// ---- B.4 updateMatrices ------------------------------------------------------------------------------
// ---- B.4 in three steps, so that two horizontally adjacent pixels can share their R1 taps -----------------------------------
struct UmCoord {
    int x1, y1;
    float fx, fy;
    bool inside;
};
__device__ __forceinline__ UmCoord um_coord(int x, int y, float dx, float dy, int w, int h) {
    UmCoord c;
    float fx = x + dx, fy = y + dy;
    c.x1 = (int)floorf(fx);
    c.y1 = (int)floorf(fy);
    c.fx = fx - c.x1;
    c.fy = fy - c.y1;
    c.inside = c.x1 >= 0 && c.y1 >= 0 && c.x1 < w - 1 && c.y1 < h - 1;
    return c;
}
// one bilinear sample, always written in this form (the compiler's multiply-add contraction is part of the result)
__device__ __forceinline__ float um_bilinear(float a00, float a01, float a10, float a11, float v00, float v01, float v10, float v11) {
    return a00 * v00 + a01 * v01 + a10 * v10 + a11 * v11;
}
// r0[5]: the five R0 planes at (x, y); s[5]: the five bilinear samples of R1 (ignored when the tap cell is outside the image)
__device__ __forceinline__ void um_finish(int x, int y, int w, int h, float dx, float dy, const float r0[5], bool inside, const float s[5],
                                          float m[5]) {
    float r2, r3, r4, r5, r6;
    if (inside) {
        r2 = s[0];
        r3 = s[1];
        r4 = (r0[2] + s[2]) * 0.5f;
        r5 = (r0[3] + s[3]) * 0.5f;
        r6 = (r0[4] + s[4]) * 0.25f;
    } else {
        r2 = r3 = 0.f;
        r4 = r0[2];
        r5 = r0[3];
        r6 = r0[4] * 0.5f;
    }
    r2 = (r0[0] - r2) * 0.5f;
    r3 = (r0[1] - r3) * 0.5f;
    r2 = r2 + (r4 * dy + r6 * dx);
    r3 = r3 + (r6 * dy + r5 * dx);
    const float scale = c_border[min(x, 5)] * c_border[min(y, 5)] * c_border[min(w - x - 1, 5)] * c_border[min(h - y - 1, 5)];
    r2 *= scale;
    r3 *= scale;
    r4 *= scale;
    r5 *= scale;
    r6 *= scale;
    m[0] = r4 * r4 + r6 * r6;
    m[1] = (r4 + r5) * r6;
    m[2] = r5 * r5 + r6 * r6;
    m[3] = r4 * r2 + r6 * r3;
    m[4] = r6 * r2 + r5 * r3;
}
__device__ __forceinline__ void um_sample(const UmCoord &c, int pitch, const Plane5 &R1, float s[5]) {
    const float a00 = (1.f - c.fx) * (1.f - c.fy), a01 = c.fx * (1.f - c.fy), a10 = (1.f - c.fx) * c.fy, a11 = c.fx * c.fy;
    const size_t j = (size_t)c.y1 * pitch + c.x1;
#pragma unroll
    for (int k = 0; k < 5; ++k) s[k] = um_bilinear(a00, a01, a10, a11, R1.p[k][j], R1.p[k][j + 1], R1.p[k][j + pitch], R1.p[k][j + pitch + 1]);
}
// r0[5] loaded by the caller (the iteration kernel fetches them at the start of a tile, long before the flow that the R1 gather
// depends on exists)
__device__ __forceinline__ void update_matrices_px_r0(int x, int y, int w, int h, int pitch, float dx, float dy, const float r0[5],
                                                      const Plane5 &R1, float m[5]) {
    const UmCoord c = um_coord(x, y, dx, dy, w, h);
    float s[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (c.inside) um_sample(c, pitch, R1, s);
    um_finish(x, y, w, h, dx, dy, r0, c.inside, s, m);
}
// Two horizontally adjacent pixels (x, y), (x + 1, y): with a smooth flow their tap cells are neighbours (same row, x1 one apart)
// and share a column, so the pair needs 6 gathers per plane instead of 8.  Same samples, same arithmetic.
__device__ __forceinline__ void update_matrices_2px_r0(int xa, int xb, int y, int w, int h, int pitch, const float dx[2], const float dy[2],
                                                       const float r0[2][5], const Plane5 &R1, float m[2][5]) {
    const UmCoord ca = um_coord(xa, y, dx[0], dy[0], w, h), cb = um_coord(xb, y, dx[1], dy[1], w, h);
    float sa[5] = {0.f, 0.f, 0.f, 0.f, 0.f}, sb[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (ca.inside && cb.inside && ca.y1 == cb.y1 && cb.x1 == ca.x1 + 1) {
        const float a00 = (1.f - ca.fx) * (1.f - ca.fy), a01 = ca.fx * (1.f - ca.fy), a10 = (1.f - ca.fx) * ca.fy, a11 = ca.fx * ca.fy;
        const float b00 = (1.f - cb.fx) * (1.f - cb.fy), b01 = cb.fx * (1.f - cb.fy), b10 = (1.f - cb.fx) * cb.fy, b11 = cb.fx * cb.fy;
        const size_t j = (size_t)ca.y1 * pitch + ca.x1;
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const float t0 = R1.p[k][j], t1 = R1.p[k][j + 1], t2 = R1.p[k][j + 2];
            const float u0 = R1.p[k][j + pitch], u1 = R1.p[k][j + pitch + 1], u2 = R1.p[k][j + pitch + 2];
            sa[k] = um_bilinear(a00, a01, a10, a11, t0, t1, u0, u1);
            sb[k] = um_bilinear(b00, b01, b10, b11, t1, t2, u1, u2);
        }
    } else {
        if (ca.inside) um_sample(ca, pitch, R1, sa);
        if (cb.inside) um_sample(cb, pitch, R1, sb);
    }
    um_finish(xa, y, w, h, dx[0], dy[0], r0[0], ca.inside, sa, m[0]);
    um_finish(xb, y, w, h, dx[1], dy[1], r0[1], cb.inside, sb, m[1]);
}

__device__ __forceinline__ void update_matrices_px(int x, int y, int w, int h, int pitch, float dx, float dy, const Plane5 &R0,
                                                   const Plane5 &R1, float m[5]) {
    const size_t o = (size_t)y * pitch + x;
    const float r0[5] = {R0.p[0][o], R0.p[1][o], R0.p[2][o], R0.p[3][o], R0.p[4][o]};
    update_matrices_px_r0(x, y, w, h, pitch, dx, dy, r0, R1, m);
}

// Several independent pairs per launch (blockIdx.z = pair): the coarse levels are far too small to fill 132 SMs and
// every kernel of the iteration is latency-bound there, so pairs are solved side by side (same idea as the TV-L1 lanes).
constexpr int kMaxFarnBatch = 8;
struct PairArgs {
    Plane5 R0, R1, M[2];
    Plane fx, fy;    // this level's flow
    Plane pfx, pfy;  // previous (coarser) level's flow; at the coarsest level with use_initial_flow, the initial flow
    int pstep;       // floats between neighbouring pixels of pfx / pfy: 1, or 2 for an initial float2 field
    float *flow_xy;
    size_t flow_pitch_bytes;
    int bound;  // > 0: the merge writes the two quantised uint8 planes instead (PairJob)
    uint8_t *qx, *qy;
    size_t q_pitch;
    float *ox, *oy;  // non-null: the merge writes the two float planes instead (PairJob::fx / fy)
    size_t o_pitch;
};
struct FarnBatchArgs {
    PairArgs p[kMaxFarnBatch];
};

__global__ void __launch_bounds__(256) k_update_matrices(const __grid_constant__ FarnBatchArgs args, int mb) {
    const PairArgs &a = args.p[blockIdx.z];
    const Plane fxp = a.fx, fyp = a.fy;
    const Plane5 R0 = a.R0, R1 = a.R1, M = a.M[mb];
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= M.w || y >= M.h) return;
    const size_t o = (size_t)y * M.pitch + x;
    float m[5];
    update_matrices_px(x, y, M.w, M.h, M.pitch, fxp.p[o], fyp.p[o], R0, R1, m);
#pragma unroll
    for (int k = 0; k < 5; ++k) M.p[k][o] = m[k];
}

// ---- B.5 fused iteration: 13x13 box mean of the 5 planes of M -> 2x2 solve -> (optionally) rebuild M ------
// GAUSS (B.7): the 13x13 Gaussian window c_gauss_win instead of the box mean; everything else is shared.
// One CTA produces a 32 x 32 tile of flow.  The (32+12) x (32+12) window of each of the five M planes is staged
// in shared memory once (index-clamped), summed vertically (centre + symmetric pairs, the reference's order) into a
// second shared buffer, then horizontally; the solve and the rebuild of M for the next iteration happen in
// registers.  Global reads of M drop from 13 vertical taps x 5 planes per column to 1.9 per output pixel and plane.
// M is double-buffered across iterations (Mout != Min): a neighbouring tile's window must still see this iteration's M.
constexpr int BW = 32;
constexpr int BH = 16;  // 512-pixel tiles (the kernel is latency-bound)
// The staged window of one M plane: (BH + 2 HALF) rows x RW columns, RW = BW + 2 HX with HX >= HALF rounded up so that the window
// starts on a 32-byte boundary of the plane row (x0 - HX, x0 a multiple of 32) and its rows are 16-byte multiples (TMA box rule).
constexpr int HX = 8;
constexpr int RW = BW + 2 * HX;
constexpr int kBoxMinBlocks = 4;  // CTAs per SM the iteration kernel is compiled for (64 registers)
constexpr int kBoxPlaneSlot = ((RW * (BH + 12) + 31) / 32) * 32;  // floats per staged window, a multiple of 128 bytes (TMA destination)

// The part of the iteration that works out of shared memory: raw = the five (BH + 2 HALF) x (BW + 2 HALF) windows of M
// (index-clamped), vs = scratch for the vertical sums.
// after_vertical() runs once the vertical sums are in `vs` and every thread is done with `raw` (the kernel asks for the
// next tile's windows there, so they land while this tile's long half — solve, gathers, rebuild — is still running).
template <int HALF, bool GAUSS, typename Hook>
__device__ __forceinline__ void box_tile_compute(const float *raw /* [5][kBoxPlaneSlot] */, float (*vs)[BH][BW + 2 * HALF], const PairArgs &a, int mb,
                                                 int rebuild, int x0, int y0, int tid, Hook after_vertical) {
    const Plane5 Mout = a.M[mb ^ 1], R0 = a.R0, R1 = a.R1;
    const Plane fxp = a.fx, fyp = a.fy;
    constexpr int sw = BW + 2 * HALF;
    const int w = Mout.w, h = Mout.h, pitch = Mout.pitch;
    // this thread's pixels in the second half of the tile: fetch their R0 values now (no dependence on the flow), so the
    // loads are in flight during the two summation passes
    constexpr int PXE = BW * BH / 256;
    const int ety = tid / (BW / PXE), etx0 = (tid % (BW / PXE)) * PXE;
    float r0pre[PXE][5];
    const int yc0 = min(y0 + ety, h - 1);
    if (rebuild) {
#pragma unroll
        for (int o = 0; o < PXE; ++o) {
            const size_t oo = (size_t)yc0 * pitch + min(x0 + etx0 + o, w - 1);
#pragma unroll
            for (int k = 0; k < 5; ++k) r0pre[o][k] = R0.p[k][oo];
        }
    }
    // vertical sums, register-blocked: one task = 4 vertically consecutive outputs of one column and plane
    // (16 window reads for 4 sums instead of 52); each sum keeps the reference's order (centre, then symmetric
    // pairs outward).  Clamped rows are materialised in the window, which equals clamping the tap's row index.
    constexpr int VG = 4;
    for (int i = tid; i < 5 * (BH / VG) * sw; i += 256) {
        const int tx = i % sw, rest = i / sw;
        const int g = rest % (BH / VG), k = rest / (BH / VG);
        float v[VG + 2 * HALF];
#pragma unroll
        for (int q = 0; q < VG + 2 * HALF; ++q) v[q] = raw[k * kBoxPlaneSlot + (g * VG + q) * RW + tx + (HX - HALF)];
#pragma unroll
        for (int o = 0; o < VG; ++o) {
            float acc;
            if constexpr (GAUSS) {
                acc = v[o + HALF] * c_gauss_win[0];
#pragma unroll
                for (int j = 1; j <= HALF; ++j) acc = acc + (v[o + HALF - j] + v[o + HALF + j]) * c_gauss_win[j];
            } else {
                acc = v[o + HALF];
#pragma unroll
                for (int j = 1; j <= HALF; ++j) acc = acc + (v[o + HALF - j] + v[o + HALF + j]);
            }
            vs[k][g * VG + o][tx] = acc;
        }
    }
    __syncthreads();
    after_vertical();
    // horizontal sums + solve + rebuild: each thread owns PX consecutive pixels of one row
    constexpr float area_inv = 1.f / (float)((1 + 2 * HALF) * (1 + 2 * HALF));
    constexpr int PX = BW * BH / 256;
    static_assert(PX == 1 || PX == 2 || PX == 4, "tile must be 256, 512 or 1024 pixels");
    static_assert((2 * HALF) % PX == 0 && (BW + 2 * HALF) % PX == 0, "vector-aligned rows");
    {
        const int ty = tid / (BW / PX), tx0 = (tid % (BW / PX)) * PX;
        const int y = y0 + ty;
        float b[PX][5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            float v[PX + 2 * HALF];
            if (PX == 4) {
#pragma unroll
                for (int q = 0; q < (PX + 2 * HALF) / 4; ++q) {
                    const float4 t = *reinterpret_cast<const float4 *>(&vs[k][ty][tx0 + 4 * q]);
                    v[4 * q] = t.x;
                    v[4 * q + 1] = t.y;
                    v[4 * q + 2] = t.z;
                    v[4 * q + 3] = t.w;
                }
            } else if (PX == 2) {
#pragma unroll
                for (int q = 0; q < (PX + 2 * HALF) / 2; ++q) {
                    const float2 t = *reinterpret_cast<const float2 *>(&vs[k][ty][tx0 + 2 * q]);
                    v[2 * q] = t.x;
                    v[2 * q + 1] = t.y;
                }
            } else {
#pragma unroll
                for (int q = 0; q < PX + 2 * HALF; ++q) v[q] = vs[k][ty][tx0 + q];
            }
#pragma unroll
            for (int o = 0; o < PX; ++o) {
                if constexpr (GAUSS) {
                    float acc = v[o + HALF] * c_gauss_win[0];
#pragma unroll
                    for (int j = 1; j <= HALF; ++j) acc = acc + (v[o + HALF - j] + v[o + HALF + j]) * c_gauss_win[j];
                    b[o][k] = acc;
                } else {
                    float acc = v[o + HALF];
#pragma unroll
                    for (int j = 1; j <= HALF; ++j) acc = acc + (v[o + HALF - j] + v[o + HALF + j]);
                    b[o][k] = acc * area_inv;
                }
            }
        }
        // all pixels' gathers are issued before any of them is consumed: coordinates are clamped into the image
        // (safe reads), only the stores are predicated
        const int yc = min(y, h - 1);
        float nfx[PX], nfy[PX], m[PX][5];
#pragma unroll
        for (int o = 0; o < PX; ++o) {
            // updateFlow: g11 = b0, g12 = b1, g22 = b2, h1 = b3, h2 = b4
            const float det_inv = f_rcp(b[o][0] * b[o][2] - b[o][1] * b[o][1] + 1e-3f);
            nfx[o] = (b[o][0] * b[o][4] - b[o][1] * b[o][3]) * det_inv;
            nfy[o] = (b[o][2] * b[o][3] - b[o][1] * b[o][4]) * det_inv;
        }
        if (rebuild) {
            if (PX == 2) {
                update_matrices_2px_r0(min(x0 + tx0, w - 1), min(x0 + tx0 + 1, w - 1), yc, w, h, pitch, nfx, nfy, r0pre, R1, m);
            } else {
#pragma unroll
                for (int o = 0; o < PX; ++o) update_matrices_px_r0(min(x0 + tx0 + o, w - 1), yc, w, h, pitch, nfx[o], nfy[o], r0pre[o], R1, m[o]);
            }
        }
#pragma unroll
        for (int o = 0; o < PX; ++o) {
            const int x = x0 + tx0 + o;
            if (x < w && y < h) {
                const size_t oo = (size_t)y * pitch + x;
                fxp.p[oo] = nfx[o];
                fyp.p[oo] = nfy[o];
                if (rebuild) {
#pragma unroll
                    for (int k = 0; k < 5; ++k) Mout.p[k][oo] = m[o][k];
                }
            }
        }
    }
}

// The iteration is a persistent kernel with TMA-staged windows: a CTA walks the tile list of the whole batch (pairs x tile
// rows x tile columns).  The five windows of a tile arrive by cp.async.bulk.tensor.2d (completion on an mbarrier, zero fill
// outside the image).  The staging buffer is free again as soon as the vertical sums are done, so the request for the NEXT
// tile's windows goes out there and the copy runs under this tile's long half (solve, the R1 gathers, rebuild of M): one
// buffer, 41 KB of shared memory, and no exposed staging loop.
// Index-clamped borders: tiles that touch the image border copy the nearest in-image entry of the window into the
// zero-filled ones (border tiles only), which reproduces index-clamped reads of M bit for bit.
template <int HALF>
struct BoxTmaSmem {
    float raw[5][kBoxPlaneSlot];
    float vs[5][BH][BW + 2 * HALF];
    unsigned long long bar;
};

template <int HALF, bool GAUSS = false>
__global__ void __launch_bounds__(256, kBoxMinBlocks) k_box_solve_update(const __grid_constant__ FarnBatchArgs args, const char *maps, int nb, int ntx, int nty,
                                                                 int mb, int rebuild) {
    constexpr int sh = BH + 2 * HALF;
    static_assert(RW * sh <= kBoxPlaneSlot && (RW * 4) % 16 == 0 && HX >= HALF, "window fits its slot, rows are 16-byte multiples");
    extern __shared__ __align__(128) unsigned char box_tma_smem[];
    BoxTmaSmem<HALF> &sm = *reinterpret_cast<BoxTmaSmem<HALF> *>(box_tma_smem);
    const int tid = threadIdx.x;
    const int per = ntx * nty, total = nb * per;
    if (tid == 0) mbar_init(&sm.bar, 1);
    __syncthreads();
    auto issue = [&](int t) {  // thread 0: the five windows of tile t
        const int z = t / per, r = t - z * per, ty = r / ntx, tx = r - ty * ntx;
        const char *m = maps + (size_t)((z * 2 + mb) * 5) * kTensorMapBytes;
        mbar_expect_tx(&sm.bar, 5u * RW * sh * (unsigned)sizeof(float));
#pragma unroll
        for (int k = 0; k < 5; ++k) tma_load_2d(sm.raw[k], m + k * kTensorMapBytes, tx * BW - HX, ty * BH - HALF, &sm.bar);
    };
    int t = blockIdx.x;
    if (t < total && tid == 0) issue(t);
    for (int i = 0; t < total; ++i, t += gridDim.x) {
        mbar_wait(&sm.bar, i & 1);
        const int z = t / per, r = t - z * per, tyi = r / ntx, txi = r - tyi * ntx;
        const PairArgs &a = args.p[z];
        const int x0 = txi * BW, y0 = tyi * BH;
        const int w = a.M[mb].w, h = a.M[mb].h;
        if (x0 < HX || y0 < HALF || x0 + BW + HX > w || y0 + BH + HALF > h) {
            for (int j = tid; j < sh * RW; j += 256) {
                const int ty = j / RW, tx = j - ty * RW;
                const int gy = y0 + ty - HALF, gx = x0 + tx - HX;
                const int cy = max(0, min(gy, h - 1)), cx = max(0, min(gx, w - 1));
                if (cy != gy || cx != gx) {
                    const int src = (cy - y0 + HALF) * RW + (cx - x0 + HX);  // an in-image entry: never written by this loop
#pragma unroll
                    for (int k = 0; k < 5; ++k) sm.raw[k][j] = sm.raw[k][src];
                }
            }
            __syncthreads();
        }
        const int tn = t + (int)gridDim.x;
        box_tile_compute<HALF, GAUSS>(&sm.raw[0][0], sm.vs, a, mb, rebuild, x0, y0, tid, [&]() {
            // every thread has passed the barrier behind the vertical sums: the staging buffer is dead
            if (tn < total && tid == 0) {
                fence_proxy_async();
                issue(tn);
            }
        });
        __syncthreads();  // vs is rewritten by the next tile's vertical sums
    }
}

// level start: flow = 0 at the coarsest level, else resize(prev) * (1/pyrScale) (B.2), both components, batched.  With
// use_initial_flow the coarsest level is resize(initial flow) * pyrScale^k the same way (first = 0, pfx / pfy the initial flow).
__global__ void __launch_bounds__(256) k_flow_init(const __grid_constant__ FarnBatchArgs args, int first, float rfx, float rfy, float mul) {
    const PairArgs &a = args.p[blockIdx.z];
    const int dx = blockIdx.x * 32 + threadIdx.x, dy = blockIdx.y * 8 + threadIdx.y;
    if (dx >= a.fx.w || dy >= a.fx.h) return;
    const size_t o = (size_t)dy * a.fx.pitch + dx;
    if (first) {
        a.fx.p[o] = 0.f;
        a.fy.p[o] = 0.f;
        return;
    }
    const Plane s1 = a.pfx, s2 = a.pfy;
    const float sx = dx * rfx, sy = dy * rfy;
    const int x1 = __float2int_rd(sx), y1 = __float2int_rd(sy);
    const int x2 = x1 + 1, y2 = y1 + 1;
    const size_t r1 = (size_t)min(y1, s1.h - 1) * s1.pitch, r2 = (size_t)min(y2, s1.h - 1) * s1.pitch;
    const int x1r = min(x1, s1.w - 1) * a.pstep, x2r = min(x2, s1.w - 1) * a.pstep;
    const float w11 = (x2 - sx) * (y2 - sy), w12 = (sx - x1) * (y2 - sy), w21 = (x2 - sx) * (sy - y1), w22 = (sx - x1) * (sy - y1);
    float o1 = 0.f, o2 = 0.f;
    o1 = o1 + s1.p[r1 + x1r] * w11;
    o1 = o1 + s1.p[r1 + x2r] * w12;
    o1 = o1 + s1.p[r2 + x1r] * w21;
    o1 = o1 + s1.p[r2 + x2r] * w22;
    o2 = o2 + s2.p[r1 + x1r] * w11;
    o2 = o2 + s2.p[r1 + x2r] * w12;
    o2 = o2 + s2.p[r2 + x1r] * w21;
    o2 = o2 + s2.p[r2 + x2r] * w22;
    a.fx.p[o] = o1 * mul;
    a.fy.p[o] = o2 * mul;
}

__global__ void __launch_bounds__(256) k_farn_merge(const __grid_constant__ FarnBatchArgs args) {
    const PairArgs &a = args.p[blockIdx.z];
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= a.fx.w || y >= a.fx.h) return;
    const float u = a.fx.p[(size_t)y * a.fx.pitch + x], v = a.fy.p[(size_t)y * a.fy.pitch + x];
    if (a.bound > 0) {  // convertFlowToImage (src/common.cpp:4-16) as the epilogue
        a.qx[(size_t)y * a.q_pitch + x] = quantise_px(u, -(double)a.bound, (double)a.bound);
        a.qy[(size_t)y * a.q_pitch + x] = quantise_px(v, -(double)a.bound, (double)a.bound);
        return;
    }
    if (a.ox) {
        const size_t d = (size_t)y * (a.o_pitch >> 2) + x;
        a.ox[d] = u;
        a.oy[d] = v;
        return;
    }
    float2 *row = reinterpret_cast<float2 *>(reinterpret_cast<char *>(a.flow_xy) + (size_t)y * a.flow_pitch_bytes);
    row[x] = make_float2(u, v);
}

struct FarnParams {
    int num_levels = 5;
    double pyr_scale = 0.5;
    int win_size = 13;
    int num_iters = 10;
    int poly_n = 5;
    double poly_sigma = 1.1;
    int use_initial_flow = 0;  // 1: each pair starts from the flow its call passes in (PairJob::init_x; DESIGN §1)
    int gaussian_window = 0;   // 1: OPTFLOW_FARNEBACK_GAUSSIAN, the 13x13 Gaussian window in every iteration (B.7)
    int fast_pyramids = 0;     // 1: fastPyramids, level images by a pyrDown chain (B.7)
};

inline int cv_round(double v) { return (int)std::nearbyint(v); }

void inv6(double a[6][6], double inv[6][6]) {
    double m[6][12];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            m[i][j] = a[i][j];
            m[i][j + 6] = i == j ? 1.0 : 0.0;
        }
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        for (int r = c + 1; r < 6; ++r)
            if (std::fabs(m[r][c]) > std::fabs(m[piv][c])) piv = r;
        if (piv != c)
            for (int j = 0; j < 12; ++j) std::swap(m[c][j], m[piv][j]);
        const double d = 1.0 / m[c][c];
        for (int j = 0; j < 12; ++j) m[c][j] *= d;
        for (int r = 0; r < 6; ++r)
            if (r != c) {
                const double f = m[r][c];
                for (int j = 0; j < 12; ++j) m[r][j] -= f * m[c][j];
            }
    }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) inv[i][j] = m[i][j + 6];
}

// B.3 constants (upstream prepareGaussian)
FarnConsts poly_constants(int n, double sigma) {
    FarnConsts c{};
    float gb[17], xgb[17], xxgb[17];
    float *g = gb + n, *xg = xgb + n, *xxg = xxgb + n;
    if (sigma < 1.19209289550781250000e-7) sigma = n * 0.3;
    double s = 0.;
    for (int x = -n; x <= n; ++x) {
        g[x] = (float)std::exp(-x * x / (2 * sigma * sigma));
        s += g[x];
    }
    s = 1. / s;
    for (int x = -n; x <= n; ++x) {
        g[x] = (float)(g[x] * s);
        xg[x] = (float)(x * g[x]);
        xxg[x] = (float)(x * x * g[x]);
    }
    double G[6][6];
    std::memset(G, 0, sizeof(G));
    for (int y = -n; y <= n; ++y)
        for (int x = -n; x <= n; ++x) {
            G[0][0] += g[y] * g[x];
            G[1][1] += g[y] * g[x] * x * x;
            G[3][3] += g[y] * g[x] * x * x * x * x;
            G[5][5] += g[y] * g[x] * x * x * y * y;
        }
    G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
    G[4][4] = G[3][3];
    G[3][4] = G[4][3] = G[5][5];
    double invG[6][6];
    inv6(G, invG);
    c.ig11 = (float)invG[1][1];
    c.ig03 = (float)invG[0][3];
    c.ig33 = (float)invG[3][3];
    c.ig55 = (float)invG[5][5];
    for (int k = 0; k <= n; ++k) {
        c.g[k] = g[k];
        c.xg[k] = xg[k];
        c.xxg[k] = xxg[k];
    }
    return c;
}

// cv::getGaussianKernel(ksize, sigma, CV_32F): fixed table for small odd ksize with sigma <= 0
GaussKernel gaussian_kernel(int ksize, double sigma) {
    GaussKernel gk{};
    gk.half = ksize / 2;
    static const float tab1[] = {1.f}, tab3[] = {0.25f, 0.5f, 0.25f}, tab5[] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    static const float tab7[] = {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f};
    const float *fixed = nullptr;
    if (ksize % 2 == 1 && ksize <= 7 && sigma <= 0) fixed = ksize == 1 ? tab1 : ksize == 3 ? tab3 : ksize == 5 ? tab5 : tab7;
    if (fixed) {
        for (int i = 0; i <= gk.half; ++i) gk.k[i] = fixed[gk.half + i];
        return gk;
    }
    const double sx = sigma > 0 ? sigma : ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8;
    const double scale2x = -0.5 / (sx * sx);
    std::vector<double> tmp(ksize);
    double sum = 0;
    for (int i = 0; i < ksize; ++i) {
        const double x = i - (ksize - 1) * 0.5;
        tmp[i] = std::exp(scale2x * x * x);
        sum += tmp[i];
    }
    sum = 1. / sum;
    for (int i = 0; i <= gk.half; ++i) gk.k[i] = (float)(tmp[gk.half + i] * sum);
    return gk;
}

class Farneback final : public FlowAlgorithm {
  public:
    Farneback(int device, int max_w, int max_h) : device_(device), max_w_(max_w), max_h_(max_h) {
        DFB_CUDA(cudaSetDevice(device_));
        pitch0_ = round_up(max_w_, 32);
        plane_elems_ = (size_t)pitch0_ * (max_h_ + 1);
        // a frame slot holds the polynomial expansion of every level (5 planes each): everything that depends on
        // one frame only, so a frame shared by two consecutive pairs is blurred / resized / expanded once.  The pyrDown
        // levels of fast_pyramids are at least as large as B.1's at every level, so slots sized for them hold both.
        LevelSet ls = levels_for(max_w_, max_h_, /*max_depth=*/true, /*fast=*/true);
        slab_.reserve(kInitialSlots * Slab::padded(ls.total_r_elems, 4) + (1 << 12));
        carve_slots(slab_, ls.total_r_elems);
        slab_.zero();
        ensure_lanes(1);
        ensure_prep_scratch(1);
        DFB_CUDA(cudaFuncSetAttribute(k_gauss_blur, cudaFuncAttributeMaxDynamicSharedMemorySize, GT * (GT + 2 * kMaxHalf) * 4));
        int sms = 0;
        DFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_));
        for (int g = 0; g < 2; ++g) {
            const auto kern = g ? k_box_solve_update<6, true> : k_box_solve_update<6>;
            DFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoxTmaSmem<6>)));
            DFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
            int per_sm = 0;
            DFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, sizeof(BoxTmaSmem<6>)));
            persistent_ctas_[g] = std::max(1, per_sm) * sms;
        }
        const GaussKernel win = gaussian_kernel(13, (double)(6.f * 0.3f));  // (float)(winSize / 2) * 0.3f, as upstream
        DFB_CUDA(cudaMemcpyToSymbol(c_gauss_win, win.k, sizeof(float) * 7));
        d_maps_.allocate(kMapBytes);
    }
    ~Farneback() override { cudaSetDevice(device_); }
    const char *name() const override { return "farn"; }
    bool set_param(const std::string &k, double v) override {
        // a refused value leaves the parameter as it was
        if (k == "num_levels") { if (!whole_in(v, 0, 5)) return false; prm_.num_levels = (int)v; }
        else if (k == "num_iters") { if (!whole_in(v, 1, INT_MAX)) return false; prm_.num_iters = (int)v; }
        else if (k == "poly_sigma") { if (!(std::isfinite(v) && v > 0)) return false; prm_.poly_sigma = v; }
        else if (k == "pyr_scale") return v == 0.5;  // level geometry and the slot layout assume the default
        else if (k == "win_size" || k == "poly_n") return (k == "win_size" ? v == 13 : v == 5);  // compiled-in stencils
        else if (k == "time_kernels") { if (!is_flag(v)) return false; time_kernels_ = v != 0; }
        else if (k == "use_initial_flow") { if (!is_flag(v)) return false; prm_.use_initial_flow = (int)v; }
        else if (k == "gaussian_window") { if (!is_flag(v)) return false; prm_.gaussian_window = (int)v; }
        else if (k == "fast_pyramids") { if (!is_flag(v)) return false; prm_.fast_pyramids = (int)v; }
        else return false;
        return true;
    }
    bool get_param(const std::string &k, double *v) const override {
        if (k == "num_levels") *v = prm_.num_levels;
        else if (k == "pyr_scale") *v = prm_.pyr_scale;
        else if (k == "win_size") *v = prm_.win_size;
        else if (k == "num_iters") *v = prm_.num_iters;
        else if (k == "poly_n") *v = prm_.poly_n;
        else if (k == "poly_sigma") *v = prm_.poly_sigma;
        else if (k == "time_kernels") *v = time_kernels_;
        else if (k == "use_initial_flow") *v = prm_.use_initial_flow;
        else if (k == "gaussian_window") *v = prm_.gaussian_window;
        else if (k == "fast_pyramids") *v = prm_.fast_pyramids;
        else return false;
        return true;
    }

    // per-frame work (B.2, B.3): u8 -> fp32, then for every level: Gaussian blur of the FULL-resolution frame,
    // bilinear resize to the level, polynomial expansion into the slot's R planes.  fast_pyramids (B.7): level 0 is the
    // fp32 frame and level k the pyrDown of level k - 1, finest first; the blur and resize kernels are not launched.
    // Slots hold a frame only within the call that prepares it, so a parameter change applies from the next call on.
    void prepare_frames(int n, const uint8_t *const *srcs, size_t pitch_bytes, int w, int h, const int *slots, cudaStream_t s) override {
        const LevelSet ls = levels_for(w, h, false, prm_.fast_pyramids);
        const int pitch_full = round_up(w, 32);
        const FarnConsts pc = poly_constants(prm_.poly_n, prm_.poly_sigma);
        for (int f0 = 0; f0 < n; f0 += kMaxPrep) {
            const int nf = std::min(kMaxPrep, n - f0);
            PrepBatch pb = prep_batch(nf);
            for (int i = 0; i < nf; ++i) pb.src[i] = srcs[f0 + i];
            launch_u8_to_f32(pb, nf, pitch_bytes, w, h, pitch_full, s);
            if (prm_.fast_pyramids) {
                PrepBatch lb = pb;  // lb.img: the level being expanded; levels k >= 1 alternate between the img and vn scratch
                for (int l = ls.n - 1; l >= 0; --l) {
                    const Level &L = ls.lv[l];
                    if (l == ls.n - 1) {
                        for (int i = 0; i < nf; ++i) lb.img[i] = pb.frame[i];
                    } else {
                        PyrBatch py{};
                        for (int i = 0; i < nf; ++i) {
                            py.src[i] = lb.img[i];
                            py.dst[i] = lb.img[i] = ((ls.n - 1 - l) & 1) ? pb.img[i] : pb.vn[i];
                        }
                        launch_pyr_down(py, nf, ls.lv[l + 1], L, s);
                    }
                    for (int i = 0; i < nf; ++i) lb.r[i] = slots_.at(slots[f0 + i]) + L.r_off;
                    launch_poly_exp(lb, nf, L, pc, s);
                }
                continue;
            }
            for (int l = 0; l < ls.n; ++l) {
                const Level &L = ls.lv[l];
                for (int i = 0; i < nf; ++i) pb.r[i] = slots_.at(slots[f0 + i]) + L.r_off;
                launch_level_image(pb, nf, w, h, pitch_full, L, s);
                launch_poly_exp(pb, nf, L, pc, s);
            }
        }
    }

    int max_concurrent_pairs(int, int) override { return kMaxFarnBatch; }

    // per-pair work (B.4, B.5): coarse -> fine, 10 fused box / solve / rebuild iterations per level
    void solve_batch(const PairJob *jobs, int count, int w, int h, cudaStream_t s) override {
        const LevelSet ls = levels_for(w, h, false, prm_.fast_pyramids);
        for (int j0 = 0; j0 < count; j0 += kMaxFarnBatch) {
            const int nb = std::min(kMaxFarnBatch, count - j0);
            ensure_lanes(nb);
            ensure_tensor_maps(ls);
            int cur = 0;
            FarnBatchArgs args{};
            for (int l = 0; l < ls.n; ++l) {
                const Level &L = ls.lv[l];
                for (int i = 0; i < nb; ++i) args.p[i] = pair_args(jobs[j0 + i], lanes_[i], ls, l, cur);
                launch_flow_init(args, nb, ls, l, s, jobs[j0].init_x != nullptr);
                int mb = 0;
                launch_update_matrices(args, nb, L, mb, s);
                pixel_iters += (uint64_t)L.w * L.h * prm_.num_iters * nb;
                // time_kernels: one timed range around the iteration launches of every level (nothing else is enqueued
                // between them); the finest level finishes the chunk's pairs
                if (time_kernels_) timer_.begin(s);
                for (int it = 0; it < prm_.num_iters; ++it) {
                    launch_iteration(args, nb, ls, l, mb, it < prm_.num_iters - 1, s);
                    mb ^= 1;
                }
                if (time_kernels_) timer_.end(s, prm_.num_iters, l == ls.n - 1 ? nb : 0);
                if (l == ls.n - 1) launch_merge(args, nb, L, s);  // last processed level is full resolution (k = 0): merge -> CV_32FC2
                cur ^= 1;
            }
        }
    }

    // Test hook (dfb_debug_run_kernel): one stage on host planes, launched by the same member functions as prepare_frames /
    // solve_batch, on the engine's own frame slots, lanes and tensor maps.
    bool debug_run(const std::string &k, const float *const *in, int n_in, float *const *out, int n_out, int w, int h, const double *scalars,
                   int n_scalars, double *) override {
        if (k.compare(0, 5, "farn_") != 0) return false;
        auto sc = [&](int i, double dflt) { return i < n_scalars ? scalars[i] : dflt; };
        auto need = [&](int ni, int no) {
            if (n_in != ni || n_out != no)
                throw std::runtime_error(k + ": expects " + std::to_string(ni) + " inputs and " + std::to_string(no) + " outputs");
        };
        auto fits = [&](int pw, int ph) {
            if (pw < 1 || ph < 1 || pw > max_w_ || ph > max_h_) throw std::runtime_error(k + ": plane size outside the handle's maximum frame size");
        };
        auto plane5 = [](const Plane5 &q, int i) { return Plane{q.p[i], q.w, q.h, q.pitch}; };
        DFB_CUDA(cudaDeviceSynchronize());  // nothing of an earlier asynchronous call may still use the slots or lanes
        const cudaStream_t s = nullptr;
        if (k == "farn_level_image") {  // in {frame (u8 values as floats)}  out {level image}  scalars {k}
            need(1, 1);
            fits(w, h);
            const LevelSet ls = levels_for(w, h, false, false);  // B.2's level image whatever fast_pyramids says
            const int lk = (int)sc(0, 0);
            if (lk < 0 || lk >= ls.n) throw std::runtime_error(k + ": level k must be in [0, " + std::to_string(ls.n) + ")");
            const Level &L = ls.lv[ls.n - 1 - lk];
            const int pitch_full = round_up(w, 32);
            PrepBatch pb = prep_batch(1);
            upload_rows(Plane{pb.frame[0], w, h, pitch_full}, in[0], 0);
            launch_level_image(pb, 1, w, h, pitch_full, L, s);
            DFB_CUDA(cudaDeviceSynchronize());
            download_rows(out[0], Plane{pb.img[0], L.w, L.h, L.pitch}, 0);
            return true;
        }
        if (k == "farn_pyr_down") {  // in {image}  out {pyrDown of it, (w + 1) / 2 x (h + 1) / 2}
            need(1, 1);
            fits(w, h);
            const Level S{w, h, round_up(w, 32), 0, 0.0, 0}, D{(w + 1) / 2, (h + 1) / 2, round_up((w + 1) / 2, 32), 0, 0.0, 0};
            PrepBatch pb = prep_batch(1);
            upload_rows(Plane{pb.frame[0], S.w, S.h, S.pitch}, in[0], 0);
            PyrBatch py{};
            py.src[0] = pb.frame[0];
            py.dst[0] = pb.img[0];
            launch_pyr_down(py, 1, S, D, s);
            DFB_CUDA(cudaDeviceSynchronize());
            download_rows(out[0], Plane{pb.img[0], D.w, D.h, D.pitch}, 0);
            return true;
        }
        if (k == "farn_poly_exp") {  // in {level image}  out {R0 .. R4}
            need(1, 5);
            fits(w, h);
            const Level L{w, h, round_up(w, 32), 0, 0.0, 0};
            PrepBatch pb = prep_batch(1);
            pb.r[0] = slots_.at(0) + L.r_off;
            upload_rows(Plane{pb.img[0], w, h, L.pitch}, in[0], 0);
            launch_poly_exp(pb, 1, L, poly_constants(prm_.poly_n, prm_.poly_sigma), s);
            DFB_CUDA(cudaDeviceSynchronize());
            const Plane5 R = r_planes(0, L);
            for (int i = 0; i < 5; ++i) download_rows(out[i], plane5(R, i), 0);
            return true;
        }
        if (k == "farn_flow_init") {  // in {fx, fy of the coarser level}  out {fx, fy}  scalars {level w, level h}
            need(2, 2);
            const int lw = (int)sc(0, 0), lh = (int)sc(1, 0);
            fits(w, h);
            fits(lw, lh);
            LevelSet ls;
            ls.n = 2;
            ls.lv[0] = Level{w, h, round_up(w, 32), 0, 0.0, 0};
            ls.lv[1] = Level{lw, lh, round_up(lw, 32), 0, 0.0, 0};
            ensure_lanes(1);
            FarnBatchArgs args{};
            args.p[0] = pair_args(PairJob{0, 1, nullptr, 0}, lanes_[0], ls, 1, 0);
            upload_rows(args.p[0].pfx, in[0], 0);
            upload_rows(args.p[0].pfy, in[1], 0);
            launch_flow_init(args, 1, ls, 1, s);
            DFB_CUDA(cudaDeviceSynchronize());
            download_rows(out[0], args.p[0].fx, 0);
            download_rows(out[1], args.p[0].fy, 0);
            return true;
        }
        if (k == "farn_initial_flow") {  // in {x, y of every pair's initial flow}  out {fx, fy of the coarsest level}  scalars {step, pitch, pairs}
            // pair i starts from rows [i * h / pairs, (i + 1) * h / pairs) of the inputs, laid out on the device as the calls pass
            // it: step 2 a float2 field, step 1 two planes, rows `pitch` floats apart (0: dense); the coarsest level of the
            // handle's num_levels comes back, stacked along the rows.  The start buffers' padding and the lanes' flow planes hold
            // NaN first; the flow planes are zero after.
            need(2, 2);
            const int step = (int)sc(0, 2), nb = (int)sc(2, 1);
            if (step != 1 && step != 2) throw std::runtime_error(k + ": step must be 1 or 2");
            if (nb < 1 || nb > kMaxFarnBatch || h % nb) throw std::runtime_error(k + ": pairs must be in [1, 8] and divide the height");
            const int ph = h / nb;
            fits(w, ph);
            const size_t row = (size_t)w * step, pitch = sc(1, 0) > 0 ? (size_t)sc(1, 0) : row;
            if (pitch < row) throw std::runtime_error(k + ": pitch smaller than a row");
            const LevelSet ls = levels_for(w, ph, false, prm_.fast_pyramids);
            const Level &L = ls.lv[0];
            ensure_slots(2 * nb);
            ensure_lanes(nb);
            const size_t pl_bytes = Slab::padded(plane_elems_, 4);
            std::vector<DeviceBuffer<float>> bufs(nb);
            FarnBatchArgs args{};
            for (int i = 0; i < nb; ++i) {
                PairJob pj{2 * i, 2 * i + 1, nullptr, 0};
                stage_initial_flow(bufs[i], pj, in[0], in[1], i * ph, w, ph, step, pitch);
                for (int b = 0; b < 2; ++b) {
                    DFB_CUDA(cudaMemset(lanes_[i].fx[b], 0xff, pl_bytes));
                    DFB_CUDA(cudaMemset(lanes_[i].fy[b], 0xff, pl_bytes));
                }
                args.p[i] = pair_args(pj, lanes_[i], ls, 0, 0);
            }
            launch_flow_init(args, nb, ls, 0, s, true);
            DFB_CUDA(cudaDeviceSynchronize());
            for (int i = 0; i < nb; ++i) {
                download_rows(out[0], args.p[i].fx, i * L.h);
                download_rows(out[1], args.p[i].fy, i * L.h);
                for (int b = 0; b < 2; ++b) {
                    DFB_CUDA(cudaMemset(lanes_[i].fx[b], 0, pl_bytes));
                    DFB_CUDA(cudaMemset(lanes_[i].fy[b], 0, pl_bytes));
                }
            }
            DFB_CUDA(cudaDeviceSynchronize());
            return true;
        }
        const bool um = k == "farn_update_matrices";
        if (!um && k != "farn_iteration") return false;
        // pair stages: every input stacks `pairs` planes of h / pairs rows along its rows, one per pair (pair i = lane i, frame
        // slots 2i / 2i + 1), so several pairs with different data run in one launch
        //   farn_update_matrices  in {fx, fy, R0 x 5, R1 x 5}  out {M0 .. M4}                 scalars {pairs}
        //   farn_iteration        in {M x 5, R0 x 5, R1 x 5}   out {fx, fy, M'0 .. M'4}        scalars {rebuild, pairs}
        const int nb = (int)sc(um ? 0 : 1, 1);
        if (nb < 1 || nb > kMaxFarnBatch || h % nb) throw std::runtime_error(k + ": pairs must be in [1, 8] and divide the height");
        const int ph = h / nb;
        um ? need(12, 5) : need(15, 7);
        fits(w, ph);
        const LevelSet ls = levels_for(w, ph, false, prm_.fast_pyramids);
        const int l = ls.n - 1;  // full resolution
        ensure_slots(2 * nb);
        ensure_lanes(nb);
        FarnBatchArgs args{};
        for (int i = 0; i < nb; ++i) {
            PairArgs &a = args.p[i] = pair_args(PairJob{2 * i, 2 * i + 1, nullptr, 0}, lanes_[i], ls, l, 0);
            const int r = i * ph;
            if (um) {
                upload_rows(a.fx, in[0], r);
                upload_rows(a.fy, in[1], r);
            }
            const float *const *rin = in + (um ? 2 : 5);
            for (int q = 0; q < 5; ++q) {
                if (!um) upload_rows(plane5(a.M[0], q), in[q], r);
                upload_rows(plane5(a.R0, q), rin[q], r);
                upload_rows(plane5(a.R1, q), rin[5 + q], r);
                fill_plane(plane5(a.M[1], q), 0);
            }
        }
        if (um) {
            launch_update_matrices(args, nb, ls.lv[l], 0, s);
        } else {
            ensure_tensor_maps(ls);
            launch_iteration(args, nb, ls, l, 0, sc(0, 1) != 0, s);
        }
        DFB_CUDA(cudaDeviceSynchronize());
        for (int i = 0; i < nb; ++i) {
            const PairArgs &a = args.p[i];
            const int r = i * ph;
            if (!um) {
                download_rows(out[0], a.fx, r);
                download_rows(out[1], a.fy, r);
            }
            for (int q = 0; q < 5; ++q) download_rows(out[(um ? 0 : 2) + q], plane5(a.M[um ? 0 : 1], q), r);
        }
        return true;
    }

  private:
    struct Level {
        int w, h, pitch, smooth;
        double sigma;
        size_t r_off;  // offset of this level's first R plane inside a slot (elements)
    };
    struct LevelSet {
        int n = 0;
        Level lv[kMaxLevels];
        size_t total_r_elems = 0;
    };
    // B.1 level list in processing order (coarsest first); fast: the same count, sizes of the pyrDown chain (B.7)
    LevelSet levels_for(int w, int h, bool max_depth, bool fast) const {
        LevelSet ls;
        const int depth = max_depth ? 5 : prm_.num_levels;
        int cropped = 0;
        double scale = 1.0;
        for (; cropped < depth; ++cropped) {
            scale *= prm_.pyr_scale;
            if (w * scale < 32 || h * scale < 32) break;
        }
        size_t off = 0;
        for (int k = cropped; k >= 0; --k) {
            scale = 1.0;
            for (int i = 0; i < k; ++i) scale *= prm_.pyr_scale;
            Level L;
            L.sigma = (1. / scale - 1) * 0.5;
            L.smooth = std::max(cv_round(L.sigma * 5) | 1, 3);
            L.w = cv_round(w * scale);
            L.h = cv_round(h * scale);
            if (fast) {
                L.w = w;
                L.h = h;
                for (int i = 0; i < k; ++i) {
                    L.w = (L.w + 1) / 2;
                    L.h = (L.h + 1) / 2;
                }
            }
            L.pitch = round_up(L.w, 32);
            L.r_off = off;
            off += 5 * (((size_t)L.pitch * (L.h + 1) + 63) & ~size_t(63));
            ls.lv[ls.n++] = L;
        }
        ls.total_r_elems = off;
        return ls;
    }
    Plane5 r_planes(int slot, const Level &L) const {
        float *base = slots_.at(slot) + L.r_off;
        const size_t pe = ((size_t)L.pitch * (L.h + 1) + 63) & ~size_t(63);
        return Plane5{{base, base + pe, base + 2 * pe, base + 3 * pe, base + 4 * pe}, L.w, L.h, L.pitch};
    }

    int device_, max_w_, max_h_, pitch0_ = 0;
    size_t plane_elems_ = 0;
    FarnParams prm_;
    Slab slab_;
    // preparation scratch of each frame of a batch: three full-resolution planes (frame, blurred rows, level image)
    std::vector<float *> prep_;
    void ensure_prep_scratch(int n) {
        while ((int)prep_.size() < n) prep_.push_back(owned_zeroed(3 * Slab::padded(plane_elems_, 4) / sizeof(float)));
    }
    // per-pair workspace: M (two buffers of five planes) and the flow of the current + previous level
    struct Lane {
        float *M[2][5] = {};
        float *fx[2] = {}, *fy[2] = {};
    };
    std::vector<Lane> lanes_;
    // TMA descriptors of the M planes: [level][lane][buffer][plane], rebuilt when the frame geometry or the lane count changes
    static constexpr size_t kMapBytes = (size_t)kMaxLevels * kMaxFarnBatch * 10 * kTensorMapBytes;
    DeviceBuffer<char> d_maps_;
    std::vector<int> maps_key_;  // lane count, then every level's size: the maps of one frame size differ with fast_pyramids
    int persistent_ctas_[2] = {132, 132};  // box, Gaussian window
    void ensure_tensor_maps(const LevelSet &ls) {
        std::vector<int> key{(int)lanes_.size()};
        for (int l = 0; l < ls.n; ++l) key.insert(key.end(), {ls.lv[l].w, ls.lv[l].h});
        if (key == maps_key_) return;
        std::vector<char> host(kMapBytes, 0);
        for (int l = 0; l < ls.n; ++l)
            for (int i = 0; i < (int)lanes_.size() && i < kMaxFarnBatch; ++i)
                for (int b = 0; b < 2; ++b)
                    for (int k = 0; k < 5; ++k)
                        encode_tensor_map_2d(host.data() + (((size_t)l * kMaxFarnBatch + i) * 10 + b * 5 + k) * kTensorMapBytes, lanes_[i].M[b][k],
                                             ls.lv[l].w, ls.lv[l].h, ls.lv[l].pitch, RW, BH + 12);
        DFB_CUDA(cudaDeviceSynchronize());  // a launch with the previous descriptors may still be running
        DFB_CUDA(cudaMemcpy(d_maps_, host.data(), host.size(), cudaMemcpyHostToDevice));
        maps_key_ = key;
    }
    int time_kernels_ = 0;
    void ensure_lanes(int n) {
        while ((int)lanes_.size() < n) {
            Lane l;
            const size_t pl = Slab::padded(plane_elems_, 4) / sizeof(float);
            float *c = owned_zeroed(14 * pl);
            for (int b = 0; b < 2; ++b)
                for (int k = 0; k < 5; ++k) {
                    l.M[b][k] = c;
                    c += pl;
                }
            for (int b = 0; b < 2; ++b) {
                l.fx[b] = c;
                c += pl;
                l.fy[b] = c;
                c += pl;
            }
            lanes_.push_back(l);
        }
    }

    // ---- launches: the one launch path of every kernel, shared by the engine and debug_run ----
    PrepBatch prep_batch(int nf) {
        ensure_prep_scratch(nf);
        PrepBatch pb{};
        const size_t pl = Slab::padded(plane_elems_, 4) / sizeof(float);
        for (int i = 0; i < nf; ++i) {
            pb.frame[i] = prep_[i];
            pb.vn[i] = prep_[i] + pl;
            pb.img[i] = prep_[i] + 2 * pl;
        }
        return pb;
    }
    void launch_u8_to_f32(const PrepBatch &pb, int nf, size_t pitch_bytes, int w, int h, int pitch_full, cudaStream_t s) {
        k_farn_u8_to_f32<<<dim3(ceil_div(w, 128), ceil_div(h, 8), nf), dim3(32, 8), 0, s>>>(pb, pitch_bytes, w, h, pitch_full);
        DFB_KERNEL_CHECK();
        ++launches;
    }
    // pb.frame (w x h, pitch_full) -> pb.img: the Gaussian blur of level L evaluated where the resize to L samples it
    void launch_level_image(const PrepBatch &pb, int nf, int w, int h, int pitch_full, const Level &L, cudaStream_t s) {
        const GaussKernel gk = gaussian_kernel(L.smooth, L.sigma);
        if (gk.half > kMaxHalf) throw std::runtime_error("farn: smoothing kernel too large");
        const float rfx = (float)(1.0 / ((double)L.w / (double)w)), rfy = (float)(1.0 / ((double)L.h / (double)h));
        if (L.w == w && L.h == h) {
            // full resolution: the resize is the identity (weights 1, 0, 0, 0), blur straight into the level image
            k_gauss_blur<<<dim3(ceil_div(w, GT), ceil_div(h, GT), nf), 256, GT * (GT + 2 * gk.half) * sizeof(float), s>>>(pb, w, h, pitch_full, gk);
            DFB_KERNEL_CHECK();
            launches += 1;
        } else {
            // vn: 2 * H_level <= h rows, fits the full-resolution scratch plane
            k_gauss_vert_rows<<<dim3(ceil_div(w, 256), 2 * L.h, nf), 256, 0, s>>>(pb, w, h, pitch_full, L.h, rfy, gk);
            DFB_KERNEL_CHECK();
            k_gauss_horz_resize<<<dim3(ceil_div(L.w, 32), ceil_div(L.h, 8), nf), dim3(32, 8), 0, s>>>(pb, w, h, pitch_full, L.w, L.h, L.pitch, rfx, rfy,
                                                                                                     gk);
            DFB_KERNEL_CHECK();
            launches += 2;
        }
    }
    // level S -> level D = pyrDown(S) of every frame of py
    void launch_pyr_down(const PyrBatch &py, int nf, const Level &S, const Level &D, cudaStream_t s) {
        k_pyr_down<<<dim3(ceil_div(D.w, 32), ceil_div(D.h, 8), nf), dim3(32, 8), 0, s>>>(py, S.w, S.h, S.pitch, D.w, D.h, D.pitch);
        DFB_KERNEL_CHECK();
        launches += 1;
    }
    // pb.img (level L) -> the five R planes at pb.r
    void launch_poly_exp(const PrepBatch &pb, int nf, const Level &L, const FarnConsts &pc, cudaStream_t s) {
        const size_t pe = ((size_t)L.pitch * (L.h + 1) + 63) & ~size_t(63);
        k_poly_exp<5><<<dim3(ceil_div(L.w, PT), ceil_div(L.h, PT), nf), 256, 0, s>>>(pb, L.w, L.h, L.pitch, pe, pc);
        DFB_KERNEL_CHECK();
        launches += 1;
    }
    // the planes of one pair at level l: R of its two frame slots, M and the flow of its lane (flow buffer `cur`, the coarser
    // level's flow in the other one)
    PairArgs pair_args(const PairJob &job, const Lane &ln, const LevelSet &ls, int l, int cur) const {
        const Level &L = ls.lv[l];
        PairArgs a{};
        a.R0 = r_planes(job.slot_a, L);
        a.R1 = r_planes(job.slot_b, L);
        for (int b = 0; b < 2; ++b) a.M[b] = Plane5{{ln.M[b][0], ln.M[b][1], ln.M[b][2], ln.M[b][3], ln.M[b][4]}, L.w, L.h, L.pitch};
        a.fx = Plane{ln.fx[cur], L.w, L.h, L.pitch};
        a.fy = Plane{ln.fy[cur], L.w, L.h, L.pitch};
        a.pstep = 1;
        if (l > 0) {
            const Level &Pv = ls.lv[l - 1];
            a.pfx = Plane{ln.fx[cur ^ 1], Pv.w, Pv.h, Pv.pitch};
            a.pfy = Plane{ln.fy[cur ^ 1], Pv.w, Pv.h, Pv.pitch};
        } else if (job.init_x) {  // the initial flow at full resolution
            const Level &F = ls.lv[ls.n - 1];
            a.pfx = Plane{const_cast<float *>(job.init_x), F.w, F.h, (int)job.init_pitch};
            a.pfy = Plane{const_cast<float *>(job.init_y), F.w, F.h, (int)job.init_pitch};
            a.pstep = job.init_step;
        }
        a.flow_xy = job.flow_xy;
        a.flow_pitch_bytes = job.flow_pitch_bytes;
        a.bound = job.bound;
        a.qx = job.qx;
        a.qy = job.qy;
        a.q_pitch = job.q_pitch;
        a.ox = job.fx;
        a.oy = job.fy;
        a.o_pitch = job.f_pitch;
        return a;
    }
    static dim3 grid8(const Level &L, int nb) { return dim3(ceil_div(L.w, 32), ceil_div(L.h, 8), nb); }
    // level start: zero at the coarsest level, else the upsampled flow of level l - 1 times 1 / pyrScale.  init (every pair of
    // the launch has an initial flow in pfx / pfy): the coarsest level is the initial flow resized to it, times pyrScale^k.
    void launch_flow_init(const FarnBatchArgs &args, int nb, const LevelSet &ls, int l, cudaStream_t s, bool init = false) {
        const Level &L = ls.lv[l];
        float rfx = 1.f, rfy = 1.f, mul = (float)(1.0 / prm_.pyr_scale);
        if (l > 0 || init) {
            const Level &S = l > 0 ? ls.lv[l - 1] : ls.lv[ls.n - 1];
            rfx = (float)(1.0 / ((double)L.w / (double)S.w));
            rfy = (float)(1.0 / ((double)L.h / (double)S.h));
        }
        if (l == 0 && init) {
            double scale = 1.0;
            for (int i = 0; i < ls.n - 1; ++i) scale *= prm_.pyr_scale;  // level k = n - 1 of B.1
            mul = (float)scale;
        }
        k_flow_init<<<grid8(L, nb), dim3(32, 8), 0, s>>>(args, l == 0 && !init, rfx, rfy, mul);
        DFB_KERNEL_CHECK();
        ++launches;
    }
    void launch_update_matrices(const FarnBatchArgs &args, int nb, const Level &L, int mb, cudaStream_t s) {
        k_update_matrices<<<grid8(L, nb), dim3(32, 8), 0, s>>>(args, mb);
        DFB_KERNEL_CHECK();
        ++launches;
    }
    // one iteration (box mean, or the Gaussian window with gaussian_window, of M[mb] -> solve -> rebuild into M[mb ^ 1]); the
    // kernel reads level l's tensor maps, which ensure_tensor_maps(ls) must have encoded
    void launch_iteration(const FarnBatchArgs &args, int nb, const LevelSet &ls, int l, int mb, int rebuild, cudaStream_t s) {
        const Level &L = ls.lv[l];
        const int ntx = ceil_div(L.w, BW), nty = ceil_div(L.h, BH);
        const int g = prm_.gaussian_window;
        const int grid = std::min(persistent_ctas_[g], ntx * nty * nb);
        const char *maps = d_maps_ + (size_t)l * kMaxFarnBatch * 10 * kTensorMapBytes;
        if (g)
            k_box_solve_update<6, true><<<grid, 256, sizeof(BoxTmaSmem<6>), s>>>(args, maps, nb, ntx, nty, mb, rebuild);
        else
            k_box_solve_update<6><<<grid, 256, sizeof(BoxTmaSmem<6>), s>>>(args, maps, nb, ntx, nty, mb, rebuild);
        DFB_KERNEL_CHECK();
        ++launches;
    }
    void launch_merge(const FarnBatchArgs &args, int nb, const Level &L, cudaStream_t s) {
        k_farn_merge<<<grid8(L, nb), dim3(32, 8), 0, s>>>(args);
        DFB_KERNEL_CHECK();
        ++launches;
    }
};

}  // namespace

std::unique_ptr<FlowAlgorithm> make_farneback(int device, int max_w, int max_h) {
    return std::unique_ptr<FlowAlgorithm>(new Farneback(device, max_w, max_h));
}

}  // namespace dfb
