// preproc.cu — the per-frame conversions the reference's decode stage applies before the hot path
// (/root/reference/src/denseflow_gpu.cpp:163-170): cvtColor(BGR2GRAY) and cv::resize(INTER_LINEAR) on uint8
// (SURVEY §8 f3).  Both are bit-exact restatements of OpenCV's CPU fixed-point arithmetic, because the flow is
// computed on these pixels: a one-level difference in the gray frame moves the flow.
//   gray   = (B*3735 + G*19235 + R*9798 + 2^14) >> 15
//   resize : 11-bit coefficients cvRound(alpha*2048) (x coefficients reset at the borders, y rows index-clamped
//            with beta kept), horizontal pass in int, vertical (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2
// The frame-extraction mode (-s=0) resizes the colour frame instead (the same arithmetic per channel) and JPEG-encodes it;
// k_bgr_to_ycc420 produces exactly the planes libjpeg would hand to its forward DCT, so only the DCT differs from imencode.
#include <cmath>
#include <vector>

#include "preproc.h"

namespace dfb {

namespace {

__global__ void __launch_bounds__(256) k_bgr_to_gray(const uint8_t *__restrict__ bgr, size_t bgr_pitch, int w, int h,
                                                     uint8_t *__restrict__ gray, size_t gray_pitch) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= w || y >= h) return;
    const uint8_t *p = bgr + (size_t)y * bgr_pitch + 3 * x;
    gray[(size_t)y * gray_pitch + x] = (uint8_t)((p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + 16384) >> 15);
}

// One INTER_LINEAR sample: source bytes i0 / i1 (the x taps, already scaled by the channel count) of the two source rows
// the y tap selects.  Shared by the gray and the colour resize so both run the same arithmetic.
__device__ __forceinline__ int resize_sample(const uint8_t *__restrict__ r0, const uint8_t *__restrict__ r1, int i0, int i1,
                                             const ResizeTap &tx, const ResizeTap &ty) {
    const int S0 = r0[i0] * tx.a0 + r0[i1] * tx.a1;
    const int S1 = r1[i0] * tx.a0 + r1[i1] * tx.a1;
    const int v = (((ty.a0 * (S0 >> 4)) >> 16) + ((ty.a1 * (S1 >> 4)) >> 16) + 2) >> 2;
    return min(max(v, 0), 255);
}

__device__ __forceinline__ const uint8_t *resize_row(const uint8_t *src, size_t src_pitch, int sh, int idx) {
    return src + (size_t)min(max(idx, 0), sh - 1) * src_pitch;
}

__global__ void __launch_bounds__(256) k_resize_u8(const uint8_t *__restrict__ src, size_t src_pitch, int sw, int sh,
                                                   uint8_t *__restrict__ dst, size_t dst_pitch, int dw, int dh,
                                                   const ResizeTap *__restrict__ xt, const ResizeTap *__restrict__ yt) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const ResizeTap tx = xt[x], ty = yt[y];
    const int x1 = min(tx.idx + 1, sw - 1);
    const uint8_t *r0 = resize_row(src, src_pitch, sh, ty.idx), *r1 = resize_row(src, src_pitch, sh, ty.idx + 1);
    dst[(size_t)y * dst_pitch + x] = (uint8_t)resize_sample(r0, r1, tx.idx, x1, tx, ty);
}

// libjpeg's rgb_ycc_convert (jccolor.c), FIX(x) = (int)(x * 65536 + 0.5); Cb and Cr carry CBCR_OFFSET + ONE_HALF - 1
__device__ __forceinline__ void bgr_to_ycc(int b, int g, int r, int &y, int &cb, int &cr) {
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// Packed BGR (sw x sh) -> cv::resize(INTER_LINEAR) to dw x dh (identity when xt == nullptr) -> JFIF YCbCr -> libjpeg's
// h2v2_downsample (jcsample.c): one thread per 2 x 2 destination block, whose chroma sample never leaves registers.
// An odd last column / row is replicated (expand_right_edge, jcsample.c; expand_bottom_edge, jcprepct.c), and the
// downsampling bias is 1 on even and 2 on odd chroma columns, restarting on every row.  Chroma columns up to c_cols are
// written (past ceil(dw / 2) only the replicated last column contributes), chroma rows up to c_rows (past ceil(dh / 2) a
// copy of the last chroma row, as expand_bottom_edge leaves the downsampled planes) and luma up to y_cols x y_rows (past
// dw x dh the last column and row replicated).
__global__ void __launch_bounds__(256) k_bgr_to_ycc420(const uint8_t *__restrict__ src, size_t src_pitch, int sw, int sh,
                                                       int dw, int dh, const ResizeTap *__restrict__ xt,
                                                       const ResizeTap *__restrict__ yt, uint8_t *__restrict__ yp, size_t y_pitch,
                                                       uint8_t *__restrict__ cbp, uint8_t *__restrict__ crp, size_t c_pitch,
                                                       int c_cols, int c_rows, int y_cols, int y_rows) {
    const int cx = blockIdx.x * 32 + threadIdx.x, cy = blockIdx.y * 8 + threadIdx.y;
    if (cx >= c_cols || cy >= c_rows) return;
    // a chroma padding row repeats the last chroma row; its luma rows all repeat row dh - 1, the second row that one reads
    const bool pad_row = cy >= (dh + 1) >> 1;
    const int cys = pad_row ? ((dh + 1) >> 1) - 1 : cy;
    int sum_cb = 0, sum_cr = 0, lum[2][2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int y = min(2 * cys + j, dh - 1);
        const uint8_t *r0, *r1 = nullptr;
        ResizeTap ty{};
        if (xt) {
            ty = yt[y];
            r0 = resize_row(src, src_pitch, sh, ty.idx);
            r1 = resize_row(src, src_pitch, sh, ty.idx + 1);
        } else {
            r0 = src + (size_t)y * src_pitch;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int x = min(2 * cx + i, dw - 1);
            int bgr[3];
            if (xt) {
                const ResizeTap tx = xt[x];
                const int i0 = 3 * tx.idx, i1 = 3 * min(tx.idx + 1, sw - 1);
#pragma unroll
                for (int c = 0; c < 3; ++c) bgr[c] = resize_sample(r0, r1, i0 + c, i1 + c, tx, ty);
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) bgr[c] = r0[3 * x + c];
            }
            int Y, Cb, Cr;
            bgr_to_ycc(bgr[0], bgr[1], bgr[2], Y, Cb, Cr);
            lum[j][i] = Y;
            sum_cb += Cb;
            sum_cr += Cr;
        }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (2 * cx + i < y_cols && 2 * cy + j < y_rows) yp[(size_t)(2 * cy + j) * y_pitch + 2 * cx + i] = (uint8_t)lum[pad_row ? 1 : j][i];
    const int bias = 1 + (cx & 1);
    cbp[(size_t)cy * c_pitch + cx] = (uint8_t)((sum_cb + bias) >> 2);
    crp[(size_t)cy * c_pitch + cx] = (uint8_t)((sum_cr + bias) >> 2);
}

// launch_pad_edges: thread t < h of plane blockIdx.y fills row t's columns [w, pw), thread h + x fills column x's rows
// [h, ph).  Both read only pixels inside the image, which nothing writes.
__global__ void __launch_bounds__(256) k_pad_edges(uint8_t *__restrict__ planes, size_t pitch, size_t plane_stride, int w, int h,
                                                   int pw, int ph) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    uint8_t *p = planes + (size_t)blockIdx.y * plane_stride;
    if (t < h) {
        uint8_t *row = p + (size_t)t * pitch;
        const uint8_t v = row[w - 1];
        for (int x = w; x < pw; ++x) row[x] = v;
    } else if (t < h + pw) {
        const int x = t - h;
        const uint8_t v = p[(size_t)(h - 1) * pitch + min(x, w - 1)];
        for (int y = h; y < ph; ++y) p[(size_t)y * pitch + x] = v;
    }
}

}  // namespace

void build_resize_taps(int dn, int sn, bool reset_at_borders, std::vector<ResizeTap> &out) {
    out.resize(dn);
    const double scale = 1.0 / ((double)dn / (double)sn);
    for (int d = 0; d < dn; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)std::floor(f);
        f -= (float)s;
        if (reset_at_borders) {
            if (s < 0) {
                f = 0.f;
                s = 0;
            }
            if (s >= sn - 1) {
                f = 0.f;
                s = sn - 1;
            }
        }
        out[d].idx = s;
        out[d].a0 = (int)std::lrintf((1.f - f) * 2048.f);
        out[d].a1 = (int)std::lrintf(f * 2048.f);
    }
}

void launch_bgr_to_gray(const uint8_t *bgr, size_t bgr_pitch, int w, int h, uint8_t *gray, size_t gray_pitch, cudaStream_t s) {
    k_bgr_to_gray<<<dim3(ceil_div(w, 32), ceil_div(h, 8)), dim3(32, 8), 0, s>>>(bgr, bgr_pitch, w, h, gray, gray_pitch);
    DFB_KERNEL_CHECK();
}

void launch_resize_u8(const uint8_t *src, size_t src_pitch, int sw, int sh, uint8_t *dst, size_t dst_pitch, int dw, int dh,
                      const ResizeTap *xt, const ResizeTap *yt, cudaStream_t s) {
    k_resize_u8<<<dim3(ceil_div(dw, 32), ceil_div(dh, 8)), dim3(32, 8), 0, s>>>(src, src_pitch, sw, sh, dst, dst_pitch, dw, dh, xt, yt);
    DFB_KERNEL_CHECK();
}

void launch_bgr_to_ycc420(const uint8_t *bgr, size_t bgr_pitch, int sw, int sh, int dw, int dh, const ResizeTap *xt, const ResizeTap *yt,
                          uint8_t *y, size_t y_pitch, uint8_t *cb, uint8_t *cr, size_t c_pitch, cudaStream_t s, YccExtent extent) {
    int c_cols = ceil_div(dw, 2), c_rows = ceil_div(dh, 2), y_cols = dw, y_rows = dh;
    if (extent != YccExtent::image) c_cols = round_up(c_cols, 8);
    if (extent == YccExtent::mcu) {
        c_rows = round_up(c_rows, 8);
        y_cols = 2 * c_cols;
        y_rows = 2 * c_rows;
    }
    k_bgr_to_ycc420<<<dim3(ceil_div(c_cols, 32), ceil_div(c_rows, 8)), dim3(32, 8), 0, s>>>(
        bgr, bgr_pitch, sw, sh, dw, dh, xt, yt, y, y_pitch, cb, cr, c_pitch, c_cols, c_rows, y_cols, y_rows);
    DFB_KERNEL_CHECK();
}

void launch_pad_edges(uint8_t *planes, size_t pitch, size_t plane_stride, int n, int w, int h, int pw, int ph, cudaStream_t s) {
    k_pad_edges<<<dim3(ceil_div(h + pw, 256), n), 256, 0, s>>>(planes, pitch, plane_stride, w, h, pw, ph);
    DFB_KERNEL_CHECK();
}

}  // namespace dfb
