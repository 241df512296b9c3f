// tvl1_math.cuh — per-pixel arithmetic of the TV-L1 inner loop, shared by the stand-alone
// kernels and the fused persistent kernel (SURVEY.md Appendix A.3; upstream
// opencv_contrib/modules/cudaoptflow/src/cuda/tvl1flow.cu estimateUKernel /
// estimateDualVariablesKernel with gamma = 0).
#pragma once

#include <cfloat>

#include "tvl1.cuh"

namespace dfb {

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

// Primal half-step (estimateU, A.3) for one pixel.  gq = tvl1_gq_from_grad(grad); div1 = div(p11,p12),
// div2 = div(p21,p22) (backward differences, p outside the image = 0).
#ifdef DFB_STRICT_FP
// Branch-free form of the reference's three-way decision: same products.
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
#else
// Every operation is an explicitly rounded IEEE fma.rn / add.rn / mul.rn: the explicit modes keep the compiler from
// contracting a product into a later sum, so the results do not depend on how ptxas schedules the code.
// rho = rho_c + I1wy*u2 + I1wx*u1 as two chained FMAs (one rounding and one instruction fewer than the reference's
// product + sum + sum; the strict build keeps the reference's association);  f = clamp(rho * q);  u' = u + f*I1w + theta*div
__device__ __forceinline__ void tvl1_primal_px(float ix, float iy, float gq, float rc, float u1o, float u2o,
                                               float div1, float div2, const Tvl1Consts &c, float &u1n,
                                               float &u2n) {
    const float rho = __fmaf_rn(ix, u1o, __fmaf_rn(iy, u2o, rc));
    const float f = fminf(fmaxf(__fmul_rn(rho, gq), -c.l_t), c.l_t);
    u1n = __fmaf_rn(c.theta, div1, __fmaf_rn(f, ix, u1o));
    u2n = __fmaf_rn(c.theta, div2, __fmaf_rn(f, iy, u2o));
}
#endif

// Dual half-step (estimateDualVariables, A.3) for one pixel, from forward differences of the NEW u (index-clamped).
#ifdef DFB_STRICT_FP
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
#else
// n = 1 + taut * sqrt.approx(ux*ux + uy*uy);  p' = (p + taut * grad u) * rcp(n)
__device__ __forceinline__ void tvl1_dual_px(float u1x, float u1y, float u2x, float u2y, float taut, float &p11,
                                             float &p12, float &p21, float &p22) {
    const float n1 = __fmaf_rn(taut, f_sqrt(__fmaf_rn(u1x, u1x, __fmul_rn(u1y, u1y))), 1.0f);
    const float n2 = __fmaf_rn(taut, f_sqrt(__fmaf_rn(u2x, u2x, __fmul_rn(u2y, u2y))), 1.0f);
    // one reciprocal for both components: 1/n1 = n2 * rcp(n1*n2), 1/n2 = n1 * rcp(n1*n2) (n >= 1: the product cannot
    // overflow or vanish).  On H100 this and two reciprocals per pixel ran at the same speed (within 0.2 %, inside the
    // run-to-run spread); this form keeps the results of earlier builds bit for bit.
    const float r = f_rcp(__fmul_rn(n1, n2));
    const float q1 = __fmul_rn(r, n2), q2 = __fmul_rn(r, n1);
    p11 = __fmul_rn(__fmaf_rn(taut, u1x, p11), q1);
    p12 = __fmul_rn(__fmaf_rn(taut, u1y, p12), q1);
    p21 = __fmul_rn(__fmaf_rn(taut, u2x, p21), q2);
    p22 = __fmul_rn(__fmaf_rn(taut, u2y, p22), q2);
}
#endif

// diff = (u1 - u1')^2 + (u2 - u2')^2 of the primal step for one pixel (fp32, as the reference's diff plane)
__device__ __forceinline__ float tvl1_diff_px(float u1o, float u2o, float u1n, float u2n) {
#ifdef DFB_STRICT_FP
    return (u1o - u1n) * (u1o - u1n) + (u2o - u2n) * (u2o - u2n);
#else
    const float e1 = __fsub_rn(u1o, u1n), e2 = __fsub_rn(u2o, u2n);
    return __fmaf_rn(e1, e1, __fmul_rn(e2, e2));
#endif
}

// Primal half-step for four horizontally adjacent pixels.
//   gq          : tvl1_gq_from_grad(grad) of the four pixels
//   p11,p21     : this row; l11,l21 = their left neighbours (0 at the image / region edge)
//   p12,p22     : this row; up12,up22 = the row above (0 at the image / region edge)
//   left_col    : pixel .x is image column 0
// div(pa,pb) = (pa(x) - pa(x-1)) + (pb(y) - pb(y-1)), summed in that order.  The reference associates image column 0
// differently: (pa + pb) - pb(y-1).  The strict build follows it there; the default build keeps the uniform form, whose
// extra rounding at that column lies within the float64 bounds the tests hold it to, rather than pay a select per row.
__device__ __forceinline__ void tvl1_primal_row(const float4 &ix, const float4 &iy, const float4 &gq, const float4 &rc,
                                                const float4 &u1o, const float4 &u2o, const float4 &p11, float l11,
                                                const float4 &p12, const float4 &up12, const float4 &p21, float l21,
                                                const float4 &p22, const float4 &up22, bool left_col, const Tvl1Consts &c,
                                                float4 &n1, float4 &n2) {
#ifdef DFB_STRICT_FP
    const float div1x = left_col ? (p11.x + p12.x) - up12.x : (p11.x - l11) + (p12.x - up12.x);
    const float div2x = left_col ? (p21.x + p22.x) - up22.x : (p21.x - l21) + (p22.x - up22.x);
#else
    (void)left_col;
    const float div1x = (p11.x - l11) + (p12.x - up12.x);
    const float div2x = (p21.x - l21) + (p22.x - up22.x);
#endif
    tvl1_primal_px(ix.x, iy.x, gq.x, rc.x, u1o.x, u2o.x, div1x, div2x, c, n1.x, n2.x);
    tvl1_primal_px(ix.y, iy.y, gq.y, rc.y, u1o.y, u2o.y, (p11.y - p11.x) + (p12.y - up12.y), (p21.y - p21.x) + (p22.y - up22.y), c, n1.y, n2.y);
    tvl1_primal_px(ix.z, iy.z, gq.z, rc.z, u1o.z, u2o.z, (p11.z - p11.y) + (p12.z - up12.z), (p21.z - p21.y) + (p22.z - up22.z), c, n1.z, n2.z);
    tvl1_primal_px(ix.w, iy.w, gq.w, rc.w, u1o.w, u2o.w, (p11.w - p11.z) + (p12.w - up12.w), (p21.w - p21.z) + (p22.w - up22.w), c, n1.w, n2.w);
}

// diff of the primal step for four pixels
__device__ __forceinline__ float4 tvl1_diff_row(const float4 &u1o, const float4 &u2o, const float4 &n1, const float4 &n2) {
    return make_float4(tvl1_diff_px(u1o.x, u2o.x, n1.x, n2.x), tvl1_diff_px(u1o.y, u2o.y, n1.y, n2.y), tvl1_diff_px(u1o.z, u2o.z, n1.z, n2.z),
                       tvl1_diff_px(u1o.w, u2o.w, n1.w, n2.w));
}

// Dual half-step for four horizontally adjacent pixels from the NEW u.
//   c1,c2 : u1,u2 of this row; d1,d2 : the row below (already index-clamped by the caller: the last image row passes
//   itself); r1,r2 : u1,u2 of the pixel right of .w (index-clamped likewise).  Pixels right of the last image column
//   inside the float4 are handled by the caller (mirrored u, or selects) before the call.
__device__ __forceinline__ void tvl1_dual_row(const float4 &c1, const float4 &c2, const float4 &d1, const float4 &d2, float r1,
                                              float r2, float taut, float4 &p11, float4 &p12, float4 &p21, float4 &p22) {
    tvl1_dual_px(c1.y - c1.x, d1.x - c1.x, c2.y - c2.x, d2.x - c2.x, taut, p11.x, p12.x, p21.x, p22.x);
    tvl1_dual_px(c1.z - c1.y, d1.y - c1.y, c2.z - c2.y, d2.y - c2.y, taut, p11.y, p12.y, p21.y, p22.y);
    tvl1_dual_px(c1.w - c1.z, d1.z - c1.z, c2.w - c2.z, d2.z - c2.z, taut, p11.z, p12.z, p21.z, p22.z);
    tvl1_dual_px(r1 - c1.w, d1.w - c1.w, r2 - c2.w, d2.w - c2.w, taut, p11.w, p12.w, p21.w, p22.w);
}

// ---- gamma > 0: the illumination field u3 with its dual planes p31, p32 (SURVEY A.8) -------------------------------------
// The gamma = 0 functions above keep their instruction sequence; these are used only by the gamma kernels.  The decision f
// is the one of tvl1_primal_px with gamma * u3 added to rho, and u3 moves by f * gamma; the convergence error stays
// (du1)^2 + (du2)^2.
#ifdef DFB_STRICT_FP
// rho = rho_c + ((I1wx*u1 + I1wy*u2) + gamma*u3), the reference's parenthesised sum
__device__ __forceinline__ void tvl1_primal_px_g(float ix, float iy, float g, float rc, float u1o, float u2o, float u3o, float div1,
                                                 float div2, float div3, const Tvl1Consts &c, float gamma, float &u1n, float &u2n,
                                                 float &u3n) {
    const float rho = rc + ((ix * u1o + iy * u2o) + gamma * u3o);
    const float thr = c.l_t * g;
    float f = g > FLT_EPSILON ? f_div(-rho, g) : 0.f;
    f = rho > thr ? -c.l_t : f;
    f = rho < -thr ? c.l_t : f;
    const float d1 = f * ix, d2 = f * iy, d3 = f * gamma;
    u1n = (u1o + d1) + c.theta * div1;
    u2n = (u2o + d2) + c.theta * div2;
    u3n = (u3o + d3) + c.theta * div3;
}
#else
// rho = rho_c + gamma*u3 + I1wy*u2 + I1wx*u1 as three chained FMAs;  u3' = u3 + f*gamma + theta*div3 like u1, u2
__device__ __forceinline__ void tvl1_primal_px_g(float ix, float iy, float gq, float rc, float u1o, float u2o, float u3o, float div1,
                                                 float div2, float div3, const Tvl1Consts &c, float gamma, float &u1n, float &u2n,
                                                 float &u3n) {
    const float rho = __fmaf_rn(ix, u1o, __fmaf_rn(iy, u2o, __fmaf_rn(gamma, u3o, rc)));
    const float f = fminf(fmaxf(__fmul_rn(rho, gq), -c.l_t), c.l_t);
    u1n = __fmaf_rn(c.theta, div1, __fmaf_rn(f, ix, u1o));
    u2n = __fmaf_rn(c.theta, div2, __fmaf_rn(f, iy, u2o));
    u3n = __fmaf_rn(c.theta, div3, __fmaf_rn(f, gamma, u3o));
}
#endif

// Dual half-step of one field (u3: p31, p32), |grad u3| exactly as tvl1_dual_px takes |grad u1|
__device__ __forceinline__ void tvl1_dual_px1(float ux, float uy, float taut, float &pa, float &pb) {
#ifdef DFB_STRICT_FP
    const float ng = 1.0f + taut * f_hypot(ux, uy);
    pa = f_div(pa + taut * ux, ng);
    pb = f_div(pb + taut * uy, ng);
#else
    const float r = f_rcp(__fmaf_rn(taut, f_sqrt(__fmaf_rn(ux, ux, __fmul_rn(uy, uy))), 1.0f));
    pa = __fmul_rn(__fmaf_rn(taut, ux, pa), r);
    pb = __fmul_rn(__fmaf_rn(taut, uy, pb), r);
#endif
}

// tvl1_primal_row with u3: u3o its four pixels, p31 / l31 / p32 / up32 as p11 / l11 / p12 / up12
__device__ __forceinline__ void tvl1_primal_row_g(const float4 &ix, const float4 &iy, const float4 &gq, const float4 &rc, const float4 &u1o,
                                                  const float4 &u2o, const float4 &u3o, const float4 &p11, float l11, const float4 &p12,
                                                  const float4 &up12, const float4 &p21, float l21, const float4 &p22, const float4 &up22,
                                                  const float4 &p31, float l31, const float4 &p32, const float4 &up32, bool left_col,
                                                  const Tvl1Consts &c, float gamma, float4 &n1, float4 &n2, float4 &n3) {
#ifdef DFB_STRICT_FP
    const float div1x = left_col ? (p11.x + p12.x) - up12.x : (p11.x - l11) + (p12.x - up12.x);
    const float div2x = left_col ? (p21.x + p22.x) - up22.x : (p21.x - l21) + (p22.x - up22.x);
    const float div3x = left_col ? (p31.x + p32.x) - up32.x : (p31.x - l31) + (p32.x - up32.x);
#else
    (void)left_col;
    const float div1x = (p11.x - l11) + (p12.x - up12.x);
    const float div2x = (p21.x - l21) + (p22.x - up22.x);
    const float div3x = (p31.x - l31) + (p32.x - up32.x);
#endif
    tvl1_primal_px_g(ix.x, iy.x, gq.x, rc.x, u1o.x, u2o.x, u3o.x, div1x, div2x, div3x, c, gamma, n1.x, n2.x, n3.x);
    tvl1_primal_px_g(ix.y, iy.y, gq.y, rc.y, u1o.y, u2o.y, u3o.y, (p11.y - p11.x) + (p12.y - up12.y), (p21.y - p21.x) + (p22.y - up22.y),
                     (p31.y - p31.x) + (p32.y - up32.y), c, gamma, n1.y, n2.y, n3.y);
    tvl1_primal_px_g(ix.z, iy.z, gq.z, rc.z, u1o.z, u2o.z, u3o.z, (p11.z - p11.y) + (p12.z - up12.z), (p21.z - p21.y) + (p22.z - up22.z),
                     (p31.z - p31.y) + (p32.z - up32.z), c, gamma, n1.z, n2.z, n3.z);
    tvl1_primal_px_g(ix.w, iy.w, gq.w, rc.w, u1o.w, u2o.w, u3o.w, (p11.w - p11.z) + (p12.w - up12.w), (p21.w - p21.z) + (p22.w - up22.w),
                     (p31.w - p31.z) + (p32.w - up32.w), c, gamma, n1.w, n2.w, n3.w);
}

// tvl1_dual_row for the one field u3 (c3: this row, d3: the row below, r3: the pixel right of .w; clamped by the caller)
__device__ __forceinline__ void tvl1_dual_row1(const float4 &c3, const float4 &d3, float r3, float taut, float4 &p31, float4 &p32) {
    tvl1_dual_px1(c3.y - c3.x, d3.x - c3.x, taut, p31.x, p32.x);
    tvl1_dual_px1(c3.z - c3.y, d3.y - c3.y, taut, p31.y, p32.y);
    tvl1_dual_px1(c3.w - c3.z, d3.z - c3.z, taut, p31.z, p32.z);
    tvl1_dual_px1(r3 - c3.w, d3.w - c3.w, taut, p31.w, p32.w);
}

// One quad of the gamma schedule (pixels x0 .. x0 + 3 of row y, x0 < W; all planes share `pitch`), shared by the stand-alone
// kernels and the fused gamma kernel so both schedules compute the same bits.  p = {p11, p12, p21, p22, p31, p32}.
// Primal, in place on u1, u2, u3 (pointwise in u, reads p only); gq = tvl1_gq_from_grad of the quad.  Returns the quad's
// sum of (du1)^2 + (du2)^2 over its image pixels when ERR.
template <bool ERR>
__device__ __forceinline__ double tvl1_gamma_primal_quad(const float *I1wx, const float *I1wy, const float4 &gq, const float *rho_c,
                                                         const float *const *p, float *u1, float *u2, float *u3, int x0, int y, int W,
                                                         int pitch, const Tvl1Consts &c, float gamma) {
    auto ld = [](const float *q) { return *reinterpret_cast<const float4 *>(q); };
    const size_t i = (size_t)y * pitch + x0;
    const float4 ix = ld(I1wx + i), iy = ld(I1wy + i), rc = ld(rho_c + i);
    const float4 a11 = ld(p[0] + i), a12 = ld(p[1] + i), a21 = ld(p[2] + i), a22 = ld(p[3] + i), a31 = ld(p[4] + i), a32 = ld(p[5] + i);
    const float4 uo1 = ld(u1 + i), uo2 = ld(u2 + i), uo3 = ld(u3 + i);
    // backward differences; p outside the image is 0 (A.3 div)
    const float l11 = x0 > 0 ? p[0][i - 1] : 0.f, l21 = x0 > 0 ? p[2][i - 1] : 0.f, l31 = x0 > 0 ? p[4][i - 1] : 0.f;
    float4 t12 = make_float4(0.f, 0.f, 0.f, 0.f), t22 = t12, t32 = t12;
    if (y > 0) {
        t12 = ld(p[1] + i - pitch);
        t22 = ld(p[3] + i - pitch);
        t32 = ld(p[5] + i - pitch);
    }
    float4 n1, n2, n3;
    tvl1_primal_row_g(ix, iy, gq, rc, uo1, uo2, uo3, a11, l11, a12, t12, a21, l21, a22, t22, a31, l31, a32, t32, x0 == 0, c, gamma, n1, n2, n3);
    *reinterpret_cast<float4 *>(u1 + i) = n1;
    *reinterpret_cast<float4 *>(u2 + i) = n2;
    *reinterpret_cast<float4 *>(u3 + i) = n3;
    double err = 0.0;
    if (ERR) {  // u3 does not enter the error
        const float4 d = tvl1_diff_row(uo1, uo2, n1, n2);
        err += (double)d.x;
        if (x0 + 1 < W) err += (double)d.y;
        if (x0 + 2 < W) err += (double)d.z;
        if (x0 + 3 < W) err += (double)d.w;
    }
    return err;
}

// Dual, in place on p (pointwise in p, reads u only): forward differences of the new u1, u2, u3, index-clamped; the last image
// column is mirrored into the pixels right of it (their results land in padding columns, never read as image data).
__device__ __forceinline__ void tvl1_gamma_dual_quad(const float *u1, const float *u2, const float *u3, float *const *p, int x0, int y, int W,
                                                     int H, int pitch, float taut) {
    auto ld = [](const float *q) { return *reinterpret_cast<const float4 *>(q); };
    const size_t i = (size_t)y * pitch + x0;
    const size_t id = (size_t)min(y + 1, H - 1) * pitch + x0;
    const size_t ir = (size_t)y * pitch + min(x0 + 4, W - 1);
    float4 c1 = ld(u1 + i), c2 = ld(u2 + i), c3 = ld(u3 + i);
    const float4 d1 = ld(u1 + id), d2 = ld(u2 + id), d3 = ld(u3 + id);
    float4 b[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) b[k] = ld(p[k] + i);
    if (x0 + 1 >= W) { c1.y = c1.x; c2.y = c2.x; c3.y = c3.x; }
    if (x0 + 2 >= W) { c1.z = c1.y; c2.z = c2.y; c3.z = c3.y; }
    if (x0 + 3 >= W) { c1.w = c1.z; c2.w = c2.z; c3.w = c3.z; }
    const bool in = x0 + 4 < W;
    tvl1_dual_row(c1, c2, d1, d2, in ? u1[ir] : c1.w, in ? u2[ir] : c2.w, taut, b[0], b[1], b[2], b[3]);
    tvl1_dual_row1(c3, d3, in ? u3[ir] : c3.w, taut, b[4], b[5]);
#pragma unroll
    for (int k = 0; k < 6; ++k) *reinterpret_cast<float4 *>(p[k] + i) = b[k];
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
