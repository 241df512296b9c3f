// tvl1_math.cuh — per-pixel arithmetic of the TV-L1 inner loop, shared by the stand-alone
// kernels and the fused persistent kernel (SURVEY.md Appendix A.3; upstream
// opencv_contrib/modules/cudaoptflow/src/cuda/tvl1flow.cu estimateUKernel /
// estimateDualVariablesKernel with gamma = 0).
#pragma once

#include <cfloat>

#include "tvl1.cuh"

namespace dfb {

// ---- fp32 pairs: two horizontally adjacent pixels, each lane an explicitly rounded IEEE operation ------------
// sm_90 has no packed fp32 instructions, so every pair operation is two scalar fma.rn / add.rn / mul.rn.  The
// explicit rounding modes keep the compiler from contracting a product into a later sum, so the results do not
// depend on how ptxas schedules the code: every place below that wants a fused multiply-add says so explicitly.
#ifndef DFB_STRICT_FP
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 lo2(const float4 &v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi2(const float4 &v) { return make_float2(v.z, v.w); }
__device__ __forceinline__ float4 cat2(float2 a, float2 b) { return make_float4(a.x, a.y, b.x, b.y); }
#endif

// ---- the "gradient" plane of the inner loop -----------------------------------------------------------------
// The reference's primal step picks d = f * (I1wx, I1wy) with f = +l_t if rho < -l_t*g, -l_t if rho > l_t*g,
// -rho/g if g > FLT_EPSILON, else 0 (A.3).  For g > eps that is exactly clamp(-rho/g, -l_t, +l_t) up to the rounding of
// the comparison at the two switch points (where both branches give the same value to an ulp), and for g <= eps it is
// sign(-rho) * l_t unless |rho| <= l_t*g < 6e-9.  The default (fast-math-like) build therefore keeps
//     q = g > eps ? -rcp(g) : -1e30        f = clamp(rho * q, -l_t, +l_t)
// (rho * -rcp(g) is bit-for-bit the product the fast-math division -rho/g expands to) and the persistent kernel stores
// q instead of g in its "grad" tile, taking the reciprocal out of the inner loop.  The strict build keeps g and the
// reference's three-way decision verbatim.
__device__ __forceinline__ float tvl1_gq_from_grad(float g) {
#ifdef DFB_STRICT_FP
    return g;
#else
    return g > FLT_EPSILON ? -f_rcp(g) : -1.0e30f;
#endif
}

#ifdef DFB_STRICT_FP
// Primal half-step for one pixel. div1 = div(p11,p12), div2 = div(p21,p22) (backward differences,
// p outside the image = 0).  Branch-free form of the reference's three-way decision: same products.
__device__ __forceinline__ void tvl1_primal_px(float ix, float iy, float g, float rc, float u1o, float u2o,
                                               float div1, float div2, const Tvl1Consts &c, float &u1n,
                                               float &u2n) {
    const float rho = rc + (ix * u1o + iy * u2o);
    const float thr = c.l_t * g;
    float f = g > FLT_EPSILON ? f_div(-rho, g) : 0.f;
    f = rho > thr ? -c.l_t : f;
    f = rho < -thr ? c.l_t : f;
    const float d1 = f * ix, d2 = f * iy;
    u1n = (u1o + d1) + c.theta * div1;
    u2n = (u2o + d2) + c.theta * div2;
}
// Dual half-step for one pixel, from forward differences of the NEW u (index-clamped).
__device__ __forceinline__ void tvl1_dual_px(float u1x, float u1y, float u2x, float u2y, float taut, float &p11,
                                             float &p12, float &p21, float &p22) {
    const float g1 = f_hypot(u1x, u1y);
    const float g2 = f_hypot(u2x, u2y);
    const float ng1 = 1.0f + taut * g1;
    const float ng2 = 1.0f + taut * g2;
    p11 = f_div(p11 + taut * u1x, ng1);
    p12 = f_div(p12 + taut * u1y, ng1);
    p21 = f_div(p21 + taut * u2x, ng2);
    p22 = f_div(p22 + taut * u2y, ng2);
}
#endif

// Primal half-step (estimateU, A.3) for four horizontally adjacent pixels.
//   gq          : tvl1_gq_from_grad(grad) of the four pixels
//   p11,p21     : this row; l11,l21 = their left neighbours (0 at the image / region edge)
//   p12,p22     : this row; up12,up22 = the row above (0 at the image / region edge)
// div(pa,pb) = (pa(x) - pa(x-1)) + (pb(y) - pb(y-1)), summed in that order.
__device__ __forceinline__ void tvl1_primal_row(const float4 &ix, const float4 &iy, const float4 &gq, const float4 &rc,
                                                const float4 &u1o, const float4 &u2o, const float4 &p11, float l11,
                                                const float4 &p12, const float4 &up12, const float4 &p21, float l21,
                                                const float4 &p22, const float4 &up22, const Tvl1Consts &c, float4 &n1,
                                                float4 &n2) {
#ifdef DFB_STRICT_FP
    tvl1_primal_px(ix.x, iy.x, gq.x, rc.x, u1o.x, u2o.x, (p11.x - l11) + (p12.x - up12.x), (p21.x - l21) + (p22.x - up22.x), c, n1.x, n2.x);
    tvl1_primal_px(ix.y, iy.y, gq.y, rc.y, u1o.y, u2o.y, (p11.y - p11.x) + (p12.y - up12.y), (p21.y - p21.x) + (p22.y - up22.y), c, n1.y, n2.y);
    tvl1_primal_px(ix.z, iy.z, gq.z, rc.z, u1o.z, u2o.z, (p11.z - p11.y) + (p12.z - up12.z), (p21.z - p21.y) + (p22.z - up22.z), c, n1.z, n2.z);
    tvl1_primal_px(ix.w, iy.w, gq.w, rc.w, u1o.w, u2o.w, (p11.w - p11.z) + (p12.w - up12.w), (p21.w - p21.z) + (p22.w - up22.w), c, n1.w, n2.w);
#else
    // rho = rho_c + I1wy*u2 + I1wx*u1;  f = clamp(rho * q);  v = u + f*(I1wx, I1wy)
    // rho as two chained FMAs (one rounding fewer than the reference's product + sum + sum, one packed instruction fewer per
    // pixel pair than mul/fma/add: +1.1 % at 1080p); the strict build keeps the reference's association
    const float2 rA = fma2(lo2(ix), lo2(u1o), fma2(lo2(iy), lo2(u2o), lo2(rc)));
    const float2 rB = fma2(hi2(ix), hi2(u1o), fma2(hi2(iy), hi2(u2o), hi2(rc)));
    float2 fA = mul2(rA, lo2(gq)), fB = mul2(rB, hi2(gq));
    const float lt = c.l_t;
    fA.x = fminf(fmaxf(fA.x, -lt), lt);
    fA.y = fminf(fmaxf(fA.y, -lt), lt);
    fB.x = fminf(fmaxf(fB.x, -lt), lt);
    fB.y = fminf(fmaxf(fB.y, -lt), lt);
    const float2 v1A = fma2(fA, lo2(ix), lo2(u1o)), v1B = fma2(fB, hi2(ix), hi2(u1o));
    const float2 v2A = fma2(fA, lo2(iy), lo2(u2o)), v2B = fma2(fB, hi2(iy), hi2(u2o));
    // divergence: horizontal differences are scalar (the shifted operand is not an aligned pair), vertical ones packed
    const float2 h1A = make_float2(p11.x - l11, p11.y - p11.x), h1B = make_float2(p11.z - p11.y, p11.w - p11.z);
    const float2 h2A = make_float2(p21.x - l21, p21.y - p21.x), h2B = make_float2(p21.z - p21.y, p21.w - p21.z);
    const float2 d1A = add2(h1A, sub2(lo2(p12), lo2(up12))), d1B = add2(h1B, sub2(hi2(p12), hi2(up12)));
    const float2 d2A = add2(h2A, sub2(lo2(p22), lo2(up22))), d2B = add2(h2B, sub2(hi2(p22), hi2(up22)));
    const float2 th = make_float2(c.theta, c.theta);
    n1 = cat2(fma2(th, d1A, v1A), fma2(th, d1B, v1B));
    n2 = cat2(fma2(th, d2A, v2A), fma2(th, d2B, v2B));
#endif
}

// diff = (u1 - u1')^2 + (u2 - u2')^2 of the primal step for four pixels (fp32, as the reference's diff plane)
__device__ __forceinline__ float4 tvl1_diff_row(const float4 &u1o, const float4 &u2o, const float4 &n1, const float4 &n2) {
    float4 d;
#ifdef DFB_STRICT_FP
    d.x = (u1o.x - n1.x) * (u1o.x - n1.x) + (u2o.x - n2.x) * (u2o.x - n2.x);
    d.y = (u1o.y - n1.y) * (u1o.y - n1.y) + (u2o.y - n2.y) * (u2o.y - n2.y);
    d.z = (u1o.z - n1.z) * (u1o.z - n1.z) + (u2o.z - n2.z) * (u2o.z - n2.z);
    d.w = (u1o.w - n1.w) * (u1o.w - n1.w) + (u2o.w - n2.w) * (u2o.w - n2.w);
#else
    const float2 e1A = sub2(lo2(u1o), lo2(n1)), e1B = sub2(hi2(u1o), hi2(n1));
    const float2 e2A = sub2(lo2(u2o), lo2(n2)), e2B = sub2(hi2(u2o), hi2(n2));
    d = cat2(fma2(e1A, e1A, mul2(e2A, e2A)), fma2(e1B, e1B, mul2(e2B, e2B)));
#endif
    return d;
}

// Dual half-step (estimateDualVariables, A.3) for four horizontally adjacent pixels from the NEW u.
//   c1,c2 : u1,u2 of this row; d1,d2 : the row below (already index-clamped by the caller: the last image row passes
//   itself); r1,r2 : u1,u2 of the pixel right of .w (index-clamped likewise).  Pixels right of the last image column
//   inside the float4 are handled by the caller (mirrored u, or selects) before the call.
__device__ __forceinline__ void tvl1_dual_row(const float4 &c1, const float4 &c2, const float4 &d1, const float4 &d2, float r1,
                                              float r2, float taut, float4 &p11, float4 &p12, float4 &p21, float4 &p22) {
#ifdef DFB_STRICT_FP
    tvl1_dual_px(c1.y - c1.x, d1.x - c1.x, c2.y - c2.x, d2.x - c2.x, taut, p11.x, p12.x, p21.x, p22.x);
    tvl1_dual_px(c1.z - c1.y, d1.y - c1.y, c2.z - c2.y, d2.y - c2.y, taut, p11.y, p12.y, p21.y, p22.y);
    tvl1_dual_px(c1.w - c1.z, d1.z - c1.z, c2.w - c2.z, d2.z - c2.z, taut, p11.z, p12.z, p21.z, p22.z);
    tvl1_dual_px(r1 - c1.w, d1.w - c1.w, r2 - c2.w, d2.w - c2.w, taut, p11.w, p12.w, p21.w, p22.w);
#else
    // forward differences: horizontal scalar, vertical packed
    const float2 x1A = make_float2(c1.y - c1.x, c1.z - c1.y), x1B = make_float2(c1.w - c1.z, r1 - c1.w);
    const float2 x2A = make_float2(c2.y - c2.x, c2.z - c2.y), x2B = make_float2(c2.w - c2.z, r2 - c2.w);
    const float2 y1A = sub2(lo2(d1), lo2(c1)), y1B = sub2(hi2(d1), hi2(c1));
    const float2 y2A = sub2(lo2(d2), lo2(c2)), y2B = sub2(hi2(d2), hi2(c2));
    // |grad u| = sqrt.approx(ux*ux + uy*uy);  1 / (1 + taut*|grad u|)
    const float2 s1A = fma2(x1A, x1A, mul2(y1A, y1A)), s1B = fma2(x1B, x1B, mul2(y1B, y1B));
    const float2 s2A = fma2(x2A, x2A, mul2(y2A, y2A)), s2B = fma2(x2B, x2B, mul2(y2B, y2B));
    const float2 t2 = make_float2(taut, taut), one = make_float2(1.0f, 1.0f);
    const float2 n1A = fma2(t2, make_float2(f_sqrt(s1A.x), f_sqrt(s1A.y)), one), n1B = fma2(t2, make_float2(f_sqrt(s1B.x), f_sqrt(s1B.y)), one);
    const float2 n2A = fma2(t2, make_float2(f_sqrt(s2A.x), f_sqrt(s2A.y)), one), n2B = fma2(t2, make_float2(f_sqrt(s2B.x), f_sqrt(s2B.y)), one);
    // one reciprocal for both components: 1/n1 = n2 * rcp(n1*n2), 1/n2 = n1 * rcp(n1*n2) (n >= 1: the product cannot
    // overflow or vanish).  The dual half-step is MUFU-bound (sqrt x2 + rcp x2 per pixel at 16 lanes per SM and clock);
    // this trades one MUFU for 1.5 packed multiplies on the idle FMA pipe at the cost of two more roundings.
#ifdef DFB_TWO_RCP
    const float2 q1A = make_float2(f_rcp(n1A.x), f_rcp(n1A.y)), q1B = make_float2(f_rcp(n1B.x), f_rcp(n1B.y));
    const float2 q2A = make_float2(f_rcp(n2A.x), f_rcp(n2A.y)), q2B = make_float2(f_rcp(n2B.x), f_rcp(n2B.y));
#else
    const float2 dA = mul2(n1A, n2A), dB = mul2(n1B, n2B);
    const float2 rA = make_float2(f_rcp(dA.x), f_rcp(dA.y)), rB = make_float2(f_rcp(dB.x), f_rcp(dB.y));
    const float2 q1A = mul2(rA, n2A), q1B = mul2(rB, n2B);
    const float2 q2A = mul2(rA, n1A), q2B = mul2(rB, n1B);
#endif
    p11 = cat2(mul2(fma2(t2, x1A, lo2(p11)), q1A), mul2(fma2(t2, x1B, hi2(p11)), q1B));
    p12 = cat2(mul2(fma2(t2, y1A, lo2(p12)), q1A), mul2(fma2(t2, y1B, hi2(p12)), q1B));
    p21 = cat2(mul2(fma2(t2, x2A, lo2(p21)), q2A), mul2(fma2(t2, x2B, hi2(p21)), q2B));
    p22 = cat2(mul2(fma2(t2, y2A, lo2(p22)), q2A), mul2(fma2(t2, y2B, hi2(p22)), q2B));
#endif
}

// Keys cubic (a = -0.5), SURVEY A.2 "Warp"
__device__ __forceinline__ float bicubic_coeff(float x) {
    x = fabsf(x);
    if (x <= 1.0f) return x * x * (1.5f * x - 2.5f) + 1.0f;
    if (x < 2.0f) return x * (x * (-0.5f * x + 2.5f) - 4.0f) + 2.0f;
    return 0.0f;
}

// A.2 "Warp (warpBackward)" for one pixel.  The reference sums taps cx = ceil(wx-2) .. floor(wx+2) (4, or 5 when wx
// is integral, in which case both end taps have weight k(+-2) = 0).  Anchored at xmin = ceil(wx-2) the distance to tap
// xmin+4 is in [2,3), so its weight is always exactly 0: a fixed 4x4 window with separable weights gives the same sums
// (tap order preserved: rows outer, columns inner).  I1 / I1x / I1y share one pitch; clamp addressing.
__device__ __forceinline__ void tvl1_warp_px(const float *__restrict__ I1, const float *I1x, const float *I1y, int W, int H, int P,
                                             int x, int y, float u1v, float u2v, float I0v, float &ix, float &iy, float &grad,
                                             float &rho_c) {
    const float wx = x + u1v, wy = y + u2v;
    const int xmin = (int)ceilf(wx - 2.0f), ymin = (int)ceilf(wy - 2.0f);
    float kx[4], ky[4];
    int cxs[4];
    size_t rows[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        kx[t] = bicubic_coeff(wx - (float)(xmin + t));
        ky[t] = bicubic_coeff(wy - (float)(ymin + t));
        cxs[t] = max(0, min(xmin + t, W - 1));
        rows[t] = (size_t)max(0, min(ymin + t, H - 1)) * P;
    }
    float sum = 0.f, sumx = 0.f, sumy = 0.f, wsum = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const float wgt = kx[b] * ky[a];
            const size_t t = rows[a] + cxs[b];
            sum = sum + wgt * __ldg(I1 + t);
            sumx = sumx + wgt * I1x[t];
            sumy = sumy + wgt * I1y[t];
            wsum = wsum + wgt;
        }
    }
    const float coeff = f_rcp(wsum);
    const float I1wv = sum * coeff;
    ix = sumx * coeff;
    iy = sumy * coeff;
    grad = ix * ix + iy * iy;
    rho_c = I1wv - ix * u1v - iy * u2v - I0v;
}

// The same warp for the persistent kernel: when the 6 x 6 neighbourhood of the 4 x 4 tap window lies inside the image (all
// but a thin border), I1x / I1y at the taps are recomputed from the I1 values themselves — 0.5f * (I1(x+1) - I1(x-1)) is exactly
// what the gradient plane holds — so the pixel costs 32 gathers instead of 48 (the phase is latency-bound).  Border pixels,
// where the gradient is taken at a CLAMPED tap coordinate, take the plane path above.  Bit-identical to tvl1_warp_px.
__device__ __forceinline__ void tvl1_warp_px_window(const float *__restrict__ I1, const float *I1x, const float *I1y, int W, int H, int P,
                                                    int x, int y, float u1v, float u2v, float I0v, float &ix, float &iy, float &grad,
                                                    float &rho_c) {
    const float wx = x + u1v, wy = y + u2v;
    const int xmin = (int)ceilf(wx - 2.0f), ymin = (int)ceilf(wy - 2.0f);
    if (xmin < 1 || ymin < 1 || xmin + 4 > W - 1 || ymin + 4 > H - 1) {
        tvl1_warp_px(I1, I1x, I1y, W, H, P, x, y, u1v, u2v, I0v, ix, iy, grad, rho_c);
        return;
    }
    float kx[4], ky[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        kx[t] = bicubic_coeff(wx - (float)(xmin + t));
        ky[t] = bicubic_coeff(wy - (float)(ymin + t));
    }
    const float *base = I1 + (size_t)(ymin - 1) * P + (xmin - 1);
    float v[6][6];
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c)
            if ((r >= 1 && r <= 4) || (c >= 1 && c <= 4)) v[r][c] = __ldg(base + (size_t)r * P + c);
    float sum = 0.f, sumx = 0.f, sumy = 0.f, wsum = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const float wgt = kx[b] * ky[a];
            sum = sum + wgt * v[a + 1][b + 1];
            sumx = sumx + wgt * (0.5f * (v[a + 1][b + 2] - v[a + 1][b]));
            sumy = sumy + wgt * (0.5f * (v[a + 2][b + 1] - v[a][b + 1]));
            wsum = wsum + wgt;
        }
    }
    const float coeff = f_rcp(wsum);
    const float I1wv = sum * coeff;
    ix = sumx * coeff;
    iy = sumy * coeff;
    grad = ix * ix + iy * iy;
    rho_c = I1wv - ix * u1v - iy * u2v - I0v;
}

}  // namespace dfb
