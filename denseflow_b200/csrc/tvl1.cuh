// tvl1.cuh — kernels of the TV-L1 path (what cv::cuda::OpticalFlowDual_TVL1::calc executes,
// /root/reference/src/denseflow_gpu.cpp:327; arithmetic per SURVEY.md Appendix A).
#pragma once

#include "common.cuh"

namespace dfb {

// ---- numeric policy -----------------------------------------------------------------------
// The reference's OpenCV is built with CUDA_FAST_MATH=ON (/root/reference/docker/Dockerfile:70):
// its divisions / hypotf are approximate.  Default build: FMA contraction on, rcp.approx /
// sqrt.approx in the inner loop.  -DDFB_STRICT_FP (+ -fmad=false): IEEE everywhere, the oracle's
// fp32 operations in the oracle's order, used by the tests to separate restatement bugs from fp
// noise.  Every stage is bit-identical to the CPU oracle; only the summation order of the
// convergence error differs (bounded in the tests).
#ifdef DFB_STRICT_FP
__device__ __forceinline__ float f_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float f_rcp(float a) { return __fdiv_rn(1.0f, a); }
// hypotf is not correctly rounded and differs between libraries: the oracle and this build both take
// (float)sqrt((double)a*a + (double)b*b) with explicit IEEE operations
__device__ __forceinline__ float f_hypot(float a, float b) {
    return __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b))));
}
#else
__device__ __forceinline__ float f_rcp(float a) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}
__device__ __forceinline__ float f_div(float a, float b) { return a * f_rcp(b); }
__device__ __forceinline__ float f_sqrt(float s) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s));
    return r;
}
__device__ __forceinline__ float f_hypot(float a, float b) { return f_sqrt(fmaf(a, a, b * b)); }
#endif

struct Tvl1Consts {
    float l_t;    // float(lambda * theta)
    float taut;   // float(tau / theta)
    float theta;  // float(theta)
};

// ---- stand-alone kernels (one launch per half-step: the reference's launch structure) -------
// the two per-frame stages for several frames of one size at once (blockIdx.z = frame): each launch is latency-bound, a
// 64-frame clip needs 5 launches instead of 320
constexpr int kMaxFrameBatch = 16;
struct FramePtrs {
    const uint8_t *src[kMaxFrameBatch];
    float *base[kMaxFrameBatch];  // the frame's pyramid slot
};
void launch_u8_to_f32_batch(const FramePtrs &fp, int n, size_t src_pitch_bytes, int w, int h, int pitch, cudaStream_t s);
// level (src_off, sw, sh, sp) -> level (dst_off, dw, dh, dp) of every frame's slot
void launch_resize_linear_batch(const FramePtrs &fp, int n, size_t src_off, int sw, int sh, int sp, size_t dst_off, int dw, int dh, int dp, float fx,
                                float fy, cudaStream_t s);
// one plane (the flow upsample and the initial flow's pyramid): the same kernel, times post_mul
void launch_resize_linear(Plane src, Plane dst, float fx, float fy, float post_mul, cudaStream_t s);
// use_initial_flow: pair i's initial field (x at x[i][y * pitch[i] + x * step[i]], y likewise) -> its lane's level-0 u1 / u2
// planes (row pitch u_pitch), for several pairs of one size at once (blockIdx.z = pair)
constexpr int kMaxInitFlows = 16;
struct InitFlows {
    const float *x[kMaxInitFlows], *y[kMaxInitFlows];
    size_t pitch[kMaxInitFlows];
    int step[kMaxInitFlows];
    float *u1[kMaxInitFlows], *u2[kMaxInitFlows];
};
void launch_split_initial_flow(const InitFlows &f, int n, int w, int h, int u_pitch, cudaStream_t s);
void launch_centered_gradient(Plane src, Plane dx, Plane dy, cudaStream_t s);
void launch_warp_backward(Plane I0, Plane I1, Plane I1x, Plane I1y, Plane u1, Plane u2, Plane I1wx, Plane I1wy,
                          Plane grad, Plane rho_c, cudaStream_t s);
// err_partials: one double per block (grid size returned by estimate_u_blocks), or nullptr
int estimate_u_blocks(int w, int h);
void launch_estimate_u(Plane I1wx, Plane I1wy, Plane grad, Plane rho_c, Plane p11, Plane p12, Plane p21, Plane p22,
                       Plane u1, Plane u2, Tvl1Consts c, double *err_partials, cudaStream_t s);
void launch_estimate_dual(Plane u1, Plane u2, Plane p11, Plane p12, Plane p21, Plane p22, Tvl1Consts c,
                          cudaStream_t s);
// gamma > 0 (SURVEY A.8): the same two half-steps with the illumination field u3; p = {p11, p12, p21, p22, p31, p32}.  The
// error partials (estimate_u_blocks of them) sum (du1)^2 + (du2)^2 only.
void launch_estimate_u_gamma(Plane I1wx, Plane I1wy, Plane grad, Plane rho_c, const Plane *p, Plane u1, Plane u2, Plane u3, Tvl1Consts c,
                             float gamma, double *err_partials, cudaStream_t s);
void launch_estimate_dual_gamma(Plane u1, Plane u2, Plane u3, const Plane *p, Tvl1Consts c, cudaStream_t s);
// fixed-order sum of n partials into *out (device or mapped host memory)
void launch_sum_partials(const double *partials, int n, double *out, cudaStream_t s);
void launch_fill(Plane dst, float v, cudaStream_t s);
// d1, d2 = the k x k median (k = 3 or 5) of u1, u2 (tvl1_median.cuh), image pixels only; out of place
void launch_median(Plane u1, Plane u2, Plane d1, Plane d2, int k, cudaStream_t s);
// the float2 field, or with fx set the two planes fx / fy (row pitch f_pitch_bytes) instead
void launch_merge_flow(Plane u1, Plane u2, float *flow_xy, size_t flow_pitch_bytes, cudaStream_t s, float *fx = nullptr,
                       float *fy = nullptr, size_t f_pitch_bytes = 0);
void launch_quantise(const float *flow_xy, size_t flow_pitch_bytes, int w, int h, int bound, uint8_t *qx, uint8_t *qy,
                     size_t q_pitch_bytes, cudaStream_t s);

}  // namespace dfb
