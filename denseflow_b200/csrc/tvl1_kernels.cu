// tvl1_kernels.cu — stand-alone sm_90a kernels of the TV-L1 path, one launch per step of
// SURVEY.md Appendix A (the reference's launch structure; the fused persistent engine lives in
// tvl1_fused.cu and reuses tvl1_math.cuh).  All planes are fp32 with 128-byte-aligned rows.
#include "tvl1.cuh"
#include "tvl1_math.cuh"

namespace dfb {

namespace {

constexpr int BX = 32, BY = 8;

inline dim3 grid2d(int w, int h, int px_per_thread_x = 1) {
    return dim3(ceil_div(w, BX * px_per_thread_x), ceil_div(h, BY));
}

// A.1: I0s[0] = float(I0), x1.0.  4 pixels per thread: one 32-bit load -> one float4 store.
__global__ void k_u8_to_f32(const uint8_t *__restrict__ src, size_t src_pitch, Plane dst) {
    const int x0 = 4 * (blockIdx.x * BX + threadIdx.x);
    const int y = blockIdx.y * BY + threadIdx.y;
    if (y >= dst.h || x0 >= dst.w) return;
    const uint8_t *row = src + (size_t)y * src_pitch;
    float4 v;
    if (x0 + 3 < dst.w && ((reinterpret_cast<uintptr_t>(row + x0) & 3) == 0)) {
        const uchar4 q = *reinterpret_cast<const uchar4 *>(row + x0);
        v = make_float4(q.x, q.y, q.z, q.w);
    } else {
        v.x = row[x0];
        v.y = x0 + 1 < dst.w ? row[x0 + 1] : 0.f;
        v.z = x0 + 2 < dst.w ? row[x0 + 2] : 0.f;
        v.w = x0 + 3 < dst.w ? row[x0 + 3] : 0.f;
    }
    *reinterpret_cast<float4 *>(dst.p + (size_t)y * dst.pitch + x0) = v;  // pitch % 32 == 0: in-bounds
}

// A.1: cudawarping resize_linear — src = dst * f (no half-pixel offset), x2/y2 reads clamped.
// post_mul folds the "u *= 1/scaleStep" multiply that follows the flow upsample (A.2 step 4).
__global__ void k_resize_linear(Plane src, Plane dst, float fx, float fy, float post_mul) {
    const int dx = blockIdx.x * BX + threadIdx.x;
    const int dy = blockIdx.y * BY + threadIdx.y;
    if (dx >= dst.w || dy >= dst.h) return;
    const float sx = dx * fx, sy = dy * fy;
    const int x1 = __float2int_rd(sx), y1 = __float2int_rd(sy);
    const int x2 = x1 + 1, y2 = y1 + 1;
    const int x1r = min(x1, src.w - 1), y1r = min(y1, src.h - 1);
    const int x2r = min(x2, src.w - 1), y2r = min(y2, src.h - 1);
    const float *r1 = src.p + (size_t)y1r * src.pitch;
    const float *r2 = src.p + (size_t)y2r * src.pitch;
    float out = 0.f;
    out = out + r1[x1r] * ((x2 - sx) * (y2 - sy));
    out = out + r1[x2r] * ((sx - x1) * (y2 - sy));
    out = out + r2[x1r] * ((x2 - sx) * (sy - y1));
    out = out + r2[x2r] * ((sx - x1) * (sy - y1));
    dst.p[(size_t)dy * dst.pitch + dx] = out * post_mul;
}

__global__ void k_u8_to_f32_batch(const __grid_constant__ FramePtrs fp, size_t src_pitch, int w, int h, int pitch) {
    const int x0 = 4 * (blockIdx.x * BX + threadIdx.x);
    const int y = blockIdx.y * BY + threadIdx.y;
    if (y >= h || x0 >= w) return;
    const uint8_t *row = fp.src[blockIdx.z] + (size_t)y * src_pitch;
    float4 v;
    if (x0 + 3 < w && ((reinterpret_cast<uintptr_t>(row + x0) & 3) == 0)) {
        const uchar4 q = *reinterpret_cast<const uchar4 *>(row + x0);
        v = make_float4(q.x, q.y, q.z, q.w);
    } else {
        v.x = row[x0];
        v.y = x0 + 1 < w ? row[x0 + 1] : 0.f;
        v.z = x0 + 2 < w ? row[x0 + 2] : 0.f;
        v.w = x0 + 3 < w ? row[x0 + 3] : 0.f;
    }
    *reinterpret_cast<float4 *>(fp.base[blockIdx.z] + (size_t)y * pitch + x0) = v;
}

// same arithmetic as k_resize_linear (post_mul = 1)
__global__ void k_resize_linear_batch(const __grid_constant__ FramePtrs fp, size_t src_off, int sw, int sh, int sp, size_t dst_off, int dw, int dh,
                                      int dp, float fx, float fy) {
    const int dx = blockIdx.x * BX + threadIdx.x;
    const int dy = blockIdx.y * BY + threadIdx.y;
    if (dx >= dw || dy >= dh) return;
    const float *src = fp.base[blockIdx.z] + src_off;
    const float sx = dx * fx, sy = dy * fy;
    const int x1 = __float2int_rd(sx), y1 = __float2int_rd(sy);
    const int x2 = x1 + 1, y2 = y1 + 1;
    const int x1r = min(x1, sw - 1), y1r = min(y1, sh - 1);
    const int x2r = min(x2, sw - 1), y2r = min(y2, sh - 1);
    const float *r1 = src + (size_t)y1r * sp;
    const float *r2 = src + (size_t)y2r * sp;
    float out = 0.f;
    out = out + r1[x1r] * ((x2 - sx) * (y2 - sy));
    out = out + r1[x2r] * ((sx - x1) * (y2 - sy));
    out = out + r2[x1r] * ((x2 - sx) * (sy - y1));
    out = out + r2[x2r] * ((sx - x1) * (sy - y1));
    fp.base[blockIdx.z][dst_off + (size_t)dy * dp + dx] = out * 1.0f;
}

// A.2 step 1: half central differences, index-clamped.
__global__ void k_centered_gradient(Plane src, Plane gx, Plane gy) {
    const int x = blockIdx.x * BX + threadIdx.x;
    const int y = blockIdx.y * BY + threadIdx.y;
    if (x >= src.w || y >= src.h) return;
    const float *row = src.p + (size_t)y * src.pitch;
    gx.p[(size_t)y * gx.pitch + x] = 0.5f * (row[min(x + 1, src.w - 1)] - row[max(x - 1, 0)]);
    gy.p[(size_t)y * gy.pitch + x] =
        0.5f * (src.p[(size_t)min(y + 1, src.h - 1) * src.pitch + x] - src.p[(size_t)max(y - 1, 0) * src.pitch + x]);
}

// A.2 "Warp (warpBackward)": weight-normalised Keys-bicubic gather of I1, I1x, I1y (clamp
// addressing, point fetches through the read-only path), grad and rho_c.  I1w itself is only an
// intermediate of rho_c and is not stored (the reference writes it; nothing reads it).
__global__ void k_warp_backward(Plane I0, Plane I1, Plane I1x, Plane I1y, Plane u1, Plane u2, Plane I1wx, Plane I1wy,
                                Plane grad, Plane rho_c) {
    const int x = blockIdx.x * BX + threadIdx.x;
    const int y = blockIdx.y * BY + threadIdx.y;
    if (x >= I0.w || y >= I0.h) return;
    const size_t i = (size_t)y * I0.pitch + x;  // all level planes share one pitch
    float ix, iy, g, rc;
    tvl1_warp_px(I1.p, I1x.p, I1y.p, I0.w, I0.h, I0.pitch, x, y, u1.p[i], u2.p[i], I0.p[i], ix, iy, g, rc);
    I1wx.p[i] = ix;
    I1wy.p[i] = iy;
    grad.p[i] = g;
    rho_c.p[i] = rc;
}

__device__ __forceinline__ float4 ld4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }

// A.3 primal (estimateU): 4 pixels per thread, float4 on all ten input planes + the two scalar
// left-neighbour taps of p11/p21 and the float4 row above of p12/p22.  48 B/px compulsory traffic.
template <bool CALC_ERROR>
__global__ void __launch_bounds__(BX *BY)
    k_estimate_u(Plane I1wx, Plane I1wy, Plane grad, Plane rho_c, Plane p11, Plane p12, Plane p21, Plane p22, Plane u1,
                 Plane u2, Tvl1Consts c, double *__restrict__ err_partials) {
    const int x0 = 4 * (blockIdx.x * BX + threadIdx.x);
    const int y = blockIdx.y * BY + threadIdx.y;
    const int W = u1.w, H = u1.h;
    double err = 0.0;
    if (y < H && x0 < W) {
        const size_t i = (size_t)y * u1.pitch + x0;
        const float4 ix = ld4(I1wx.p + i), iy = ld4(I1wy.p + i), g = ld4(grad.p + i), rc = ld4(rho_c.p + i);
        const float4 a11 = ld4(p11.p + i), a12 = ld4(p12.p + i), a21 = ld4(p21.p + i), a22 = ld4(p22.p + i);
        const float4 uo1 = ld4(u1.p + i), uo2 = ld4(u2.p + i);
        // backward differences; p outside the image is 0 (A.3 div)
        const float l11 = x0 > 0 ? p11.p[i - 1] : 0.f;
        const float l21 = x0 > 0 ? p21.p[i - 1] : 0.f;
        float4 t12 = make_float4(0.f, 0.f, 0.f, 0.f), t22 = t12;
        if (y > 0) {
            t12 = ld4(p12.p + i - p12.pitch);
            t22 = ld4(p22.p + i - p22.pitch);
        }
        float4 n1, n2;
        const float4 gq = make_float4(tvl1_gq_from_grad(g.x), tvl1_gq_from_grad(g.y), tvl1_gq_from_grad(g.z), tvl1_gq_from_grad(g.w));
        tvl1_primal_row(ix, iy, gq, rc, uo1, uo2, a11, l11, a12, t12, a21, l21, a22, t22, c, n1, n2);
        st4(u1.p + i, n1);
        st4(u2.p + i, n2);
        if (CALC_ERROR) {
            // diff = (u1-u1')^2 + (u2-u2')^2 in fp32 per pixel, accumulated in double (cuda::sum)
            const float4 d = tvl1_diff_row(uo1, uo2, n1, n2);
            err += (double)d.x;
            if (x0 + 1 < W) err += (double)d.y;
            if (x0 + 2 < W) err += (double)d.z;
            if (x0 + 3 < W) err += (double)d.w;
        }
    }
    if (CALC_ERROR) {
        __shared__ double warp_sums[BY];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) err += __shfl_xor_sync(0xffffffffu, err, o);
        if (threadIdx.x == 0) warp_sums[threadIdx.y] = err;
        __syncthreads();
        if (threadIdx.x == 0 && threadIdx.y == 0) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < BY; ++k) s += warp_sums[k];
            err_partials[blockIdx.y * gridDim.x + blockIdx.x] = s;
        }
    }
}

// A.3 dual (estimateDualVariables): forward differences of the new u, index-clamped.  40 B/px.
__global__ void __launch_bounds__(BX *BY)
    k_estimate_dual(Plane u1, Plane u2, Plane p11, Plane p12, Plane p21, Plane p22, Tvl1Consts c) {
    const int x0 = 4 * (blockIdx.x * BX + threadIdx.x);
    const int y = blockIdx.y * BY + threadIdx.y;
    const int W = u1.w, H = u1.h;
    if (y >= H || x0 >= W) return;
    const size_t i = (size_t)y * u1.pitch + x0;
    const float4 a1 = ld4(u1.p + i), a2 = ld4(u2.p + i);
    const size_t id = (size_t)min(y + 1, H - 1) * u1.pitch + x0;
    const float4 d1 = ld4(u1.p + id), d2 = ld4(u2.p + id);
    // right neighbour of the 4th pixel (index-clamped at the image edge)
    const int xr = min(x0 + 4, W - 1);
    const float r1 = u1.p[(size_t)y * u1.pitch + xr], r2 = u2.p[(size_t)y * u2.pitch + xr];
    float4 b11 = ld4(p11.p + i), b12 = ld4(p12.p + i), b21 = ld4(p21.p + i), b22 = ld4(p22.p + i);
    // u(x+1) - u(x) with u(x+1) = u(x) when x == W-1: mirror the last image column into the pixels right of it (their own
    // results land in the padding columns and are never read as image data)
    float4 c1 = a1, c2 = a2;
    if (x0 + 1 >= W) { c1.y = c1.x; c2.y = c2.x; }
    if (x0 + 2 >= W) { c1.z = c1.y; c2.z = c2.y; }
    if (x0 + 3 >= W) { c1.w = c1.z; c2.w = c2.z; }
    tvl1_dual_row(c1, c2, d1, d2, x0 + 4 < W ? r1 : c1.w, x0 + 4 < W ? r2 : c2.w, c.taut, b11, b12, b21, b22);
    st4(p11.p + i, b11);
    st4(p12.p + i, b12);
    st4(p21.p + i, b21);
    st4(p22.p + i, b22);
}

__global__ void k_sum_partials(const double *__restrict__ partials, int n, double *out) {
    // fixed-order tree: thread t sums partials[t], [t+256], ...; then a fixed shuffle/smem tree
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
    __shared__ double sm[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += sm[k];
        *out = t;
    }
}

__global__ void k_fill(Plane dst, float v) {
    const int x0 = 4 * (blockIdx.x * BX + threadIdx.x);
    const int y = blockIdx.y * BY + threadIdx.y;
    if (y >= dst.h || x0 >= dst.pitch) return;
    st4(dst.p + (size_t)y * dst.pitch + x0, make_float4(v, v, v, v));
}

// A.5: merge(u1, u2) -> CV_32FC2
__global__ void k_merge_flow(Plane u1, Plane u2, float *flow, size_t flow_pitch_bytes) {
    const int x = blockIdx.x * BX + threadIdx.x;
    const int y = blockIdx.y * BY + threadIdx.y;
    if (x >= u1.w || y >= u1.h) return;
    float2 *row = reinterpret_cast<float2 *>(reinterpret_cast<char *>(flow) + (size_t)y * flow_pitch_bytes);
    row[x] = make_float2(u1.p[(size_t)y * u1.pitch + x], u2.p[(size_t)y * u2.pitch + x]);
}

// convertFlowToImage, /root/reference/src/common.cpp:4-16 (quantise_px, common.cuh)
__global__ void k_quantise(const float *flow, size_t flow_pitch_bytes, int w, int h, double L, double H, uint8_t *qx,
                           uint8_t *qy, size_t q_pitch) {
    const int x = blockIdx.x * BX + threadIdx.x;
    const int y = blockIdx.y * BY + threadIdx.y;
    if (x >= w || y >= h) return;
    const float2 f = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(flow) + (size_t)y * flow_pitch_bytes)[x];
    qx[(size_t)y * q_pitch + x] = quantise_px(f.x, L, H);
    qy[(size_t)y * q_pitch + x] = quantise_px(f.y, L, H);
}

}  // namespace

void launch_u8_to_f32(const uint8_t *src, size_t src_pitch_bytes, Plane dst, cudaStream_t s) {
    k_u8_to_f32<<<grid2d(dst.w, dst.h, 4), dim3(BX, BY), 0, s>>>(src, src_pitch_bytes, dst);
    DFB_KERNEL_CHECK();
}
void launch_u8_to_f32_batch(const FramePtrs &fp, int n, size_t src_pitch_bytes, int w, int h, int pitch, cudaStream_t s) {
    const dim3 g = grid2d(w, h, 4);
    k_u8_to_f32_batch<<<dim3(g.x, g.y, n), dim3(BX, BY), 0, s>>>(fp, src_pitch_bytes, w, h, pitch);
    DFB_KERNEL_CHECK();
}
void launch_resize_linear_batch(const FramePtrs &fp, int n, size_t src_off, int sw, int sh, int sp, size_t dst_off, int dw, int dh, int dp, float fx,
                                float fy, cudaStream_t s) {
    const dim3 g = grid2d(dw, dh);
    k_resize_linear_batch<<<dim3(g.x, g.y, n), dim3(BX, BY), 0, s>>>(fp, src_off, sw, sh, sp, dst_off, dw, dh, dp, fx, fy);
    DFB_KERNEL_CHECK();
}
void launch_resize_linear(Plane src, Plane dst, float fx, float fy, float post_mul, cudaStream_t s) {
    k_resize_linear<<<grid2d(dst.w, dst.h), dim3(BX, BY), 0, s>>>(src, dst, fx, fy, post_mul);
    DFB_KERNEL_CHECK();
}
void launch_centered_gradient(Plane src, Plane dx, Plane dy, cudaStream_t s) {
    k_centered_gradient<<<grid2d(src.w, src.h), dim3(BX, BY), 0, s>>>(src, dx, dy);
    DFB_KERNEL_CHECK();
}
void launch_warp_backward(Plane I0, Plane I1, Plane I1x, Plane I1y, Plane u1, Plane u2, Plane I1wx, Plane I1wy,
                          Plane grad, Plane rho_c, cudaStream_t s) {
    k_warp_backward<<<grid2d(I0.w, I0.h), dim3(BX, BY), 0, s>>>(I0, I1, I1x, I1y, u1, u2, I1wx, I1wy, grad, rho_c);
    DFB_KERNEL_CHECK();
}
int estimate_u_blocks(int w, int h) {
    const dim3 g = grid2d(w, h, 4);
    return (int)(g.x * g.y);
}
void launch_estimate_u(Plane I1wx, Plane I1wy, Plane grad, Plane rho_c, Plane p11, Plane p12, Plane p21, Plane p22,
                       Plane u1, Plane u2, Tvl1Consts c, double *err_partials, cudaStream_t s) {
    const dim3 g = grid2d(u1.w, u1.h, 4);
    if (err_partials)
        k_estimate_u<true><<<g, dim3(BX, BY), 0, s>>>(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, u1, u2, c, err_partials);
    else
        k_estimate_u<false><<<g, dim3(BX, BY), 0, s>>>(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, u1, u2, c, nullptr);
    DFB_KERNEL_CHECK();
}
void launch_estimate_dual(Plane u1, Plane u2, Plane p11, Plane p12, Plane p21, Plane p22, Tvl1Consts c,
                          cudaStream_t s) {
    k_estimate_dual<<<grid2d(u1.w, u1.h, 4), dim3(BX, BY), 0, s>>>(u1, u2, p11, p12, p21, p22, c);
    DFB_KERNEL_CHECK();
}
void launch_sum_partials(const double *partials, int n, double *out, cudaStream_t s) {
    k_sum_partials<<<1, 256, 0, s>>>(partials, n, out);
    DFB_KERNEL_CHECK();
}
void launch_fill(Plane dst, float v, cudaStream_t s) {
    k_fill<<<dim3(ceil_div(dst.pitch, BX * 4), ceil_div(dst.h, BY)), dim3(BX, BY), 0, s>>>(dst, v);
    DFB_KERNEL_CHECK();
}
void launch_merge_flow(Plane u1, Plane u2, float *flow_xy, size_t flow_pitch_bytes, cudaStream_t s) {
    k_merge_flow<<<grid2d(u1.w, u1.h), dim3(BX, BY), 0, s>>>(u1, u2, flow_xy, flow_pitch_bytes);
    DFB_KERNEL_CHECK();
}
void launch_quantise(const float *flow_xy, size_t flow_pitch_bytes, int w, int h, int bound, uint8_t *qx, uint8_t *qy,
                     size_t q_pitch_bytes, cudaStream_t s) {
    k_quantise<<<grid2d(w, h), dim3(BX, BY), 0, s>>>(flow_xy, flow_pitch_bytes, w, h, -(double)bound, (double)bound, qx,
                                                     qy, q_pitch_bytes);
    DFB_KERNEL_CHECK();
}

}  // namespace dfb
