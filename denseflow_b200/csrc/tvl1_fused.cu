// tvl1_fused.cu — the persistent fused TV-L1 pair kernel for sm_90a.
//
// One cooperative launch computes a whole flow field: everything procOneScale does for every
// scale of cv::cuda::OpticalFlowDual_TVL1::calc (/root/reference/src/denseflow_gpu.cpp:327;
// SURVEY.md Appendix A.2 - A.5) — centred gradients, 5 bicubic warps per scale, the primal/dual
// inner loop with its data-dependent length, the flow upsampling between scales and the final
// merge — with the A.4 convergence state machine evaluated on the device.  The reference needs
// ~2 000 launches and a host sync per convergence check for the same work.
//
// Inner loop (the hot part).  The image is cut into 128 x 64 tiles.  A CTA of 16 warps owns one tile
// at a time: lane l of warp q owns pixels x = 4l..4l+3 of rows 4q..4q+3.  The four dual planes
// (p11,p12,p21,p22) live in registers; u1,u2 and the four per-warp constants (I1wx,I1wy,grad,rho_c)
// live in shared memory (192 KB), staged there by TMA (cp.async.bulk.tensor.2d + mbarrier, zero
// fill outside the image) while the threads load the dual planes.  Horizontal neighbours come
// from warp shuffles, vertical neighbours from the thread's own rows, the shared u tile, or a
// one-row shared-memory exchange of p12/p22 between adjacent warps.  k primal+dual iterations run
// on chip per tile visit (halo = k, the valid region shrinks by one pixel per iteration, exactly
// preserving the reference's Jacobi ordering: dual sees the fully updated u, the next primal the
// fully updated p), then the interior is written to the other half of a ping-pong pair.
// Compulsory HBM traffic is 64 B/px per k iterations instead of 88 B/px per iteration.
//
// Several independent pairs ("lanes") share one launch: lane i runs on CTAs [i*G, (i+1)*G) with its
// own workspace, barrier words and TMA descriptors, so the coarse scales (fewer tiles than SMs)
// do not leave SMs idle.
//
// Grid-wide ordering uses a monotonically counting barrier in global memory per lane (all CTAs are
// co-resident: cooperative launch).  The convergence error is reduced in a fixed order
// (per-CTA partial -> every CTA sums all partials identically), so every CTA takes the same
// branch of the A.4 state machine and results are run-to-run deterministic.
#include <cfloat>
#include <cstring>


#include <mutex>

#include "tma.cuh"
#include "tvl1_fused.cuh"
#include "tvl1_math.cuh"

namespace dfb {

namespace {

#ifndef DFB_FUSED_THREADS
#define DFB_FUSED_THREADS 512
#endif
constexpr int kThreads = DFB_FUSED_THREADS;
constexpr int kWarps = kThreads / 32;
constexpr int kPartialSet = 256;  // stride between the two sets of per-CTA convergence partials (>= CTAs per lane)
#ifndef DFB_FUSED_RPT
#define DFB_FUSED_RPT 4
#endif
constexpr int RPT = DFB_FUSED_RPT;  // rows per thread
constexpr int TW = 128;           // tile width  = 32 lanes x 4 px
constexpr int TH = kWarps * RPT;  // tile height = 64
constexpr int kConstPlane = TW * TH;

struct Smem {
    float consts[4][kConstPlane];  // I1wx, I1wy, grad, rho_c of the current tile (thread-private slots)
    float u[2][kConstPlane];       // u1, u2 of the current tile: written by the owning thread in the primal step,
                                   // read by the row above / the lane to the left in the dual step
    float p_bot[2][kWarps][TW];    // row 3 of every warp's p12/p22 (read by the warp below as "up")
    double red[kWarps];
    double bcast[4];
    int ibcast[4];
    unsigned long long prof[32];
    int prog[kWarps];  // per-warp progress counters of the tile loop (see process_tile)
    unsigned long long tma_bar;  // mbarrier the TMA tile loads complete on
    FusedJob job;                // this lane's job description (copied from the device-memory ring at kernel start)
};

__device__ __forceinline__ float4 ld_cg4(const float *p) { return __ldcg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// ---- grid barrier ---------------------------------------------------------------------------
// sync[0] counts arrivals monotonically: barrier number b of a lane completes when it reaches b * G
// (G = CTAs in the lane's group).
// bar.sync orders the CTA's writes before thread 0's gpu-scope fence + atomic (release); the
// fence after the spin makes other CTAs' writes visible and invalidates this SM's L1.
__device__ __noinline__ void barrier_stalled(FusedHostCtl *ctl, unsigned epoch, unsigned v, int G) {
    volatile unsigned *st = ctl->stall;
    st[1] = blockIdx.x;
    st[2] = epoch;
    st[3] = v;
    st[4] = (unsigned)G;
    st[5] = blockIdx.x / (unsigned)G;
    __threadfence_system();
    st[0] = 1;
    __threadfence_system();
    __trap();
}
__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned &epoch, int G, FusedHostCtl *ctl) {
    __syncthreads();
    if (threadIdx.x == 0) {
        epoch += G;
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned v, polls = 0;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            // watchdog: counts polls, not wall time — a context that is switched out (time-sliced GPU) does not age
            if (++polls == kFusedStallPolls) barrier_stalled(ctl, epoch, v, G);
        } while ((int)(v - epoch) < 0);
        __threadfence();
    }
    __syncthreads();
}

// ---- pixel-parallel phases (grid-stride over the level) --------------------------------------
__device__ __forceinline__ void phase_level_start(const int G, const int bid, const FusedJob &job, const FusedLevel &L, bool coarsest) {
    const int W = L.w, H = L.h, P = L.pitch;
    const int total = H * (P >> 2);
    for (int i = bid * kThreads + threadIdx.x; i < total; i += G * kThreads) {
        const int y = i / (P >> 2), x0 = (i - y * (P >> 2)) << 2;
        const size_t o = (size_t)y * P + x0;
        // A.2 step 2: p = 0 once per scale; A.2: u = 0 at the coarsest scale
        st4(job.p[0][0] + o, zero4());
        st4(job.p[0][1] + o, zero4());
        st4(job.p[0][2] + o, zero4());
        st4(job.p[0][3] + o, zero4());
        if (coarsest) {
            st4(L.u1[0] + o, zero4());
            st4(L.u2[0] + o, zero4());
        }
        // A.2 step 1: centred gradient of I1, index-clamped
        if (x0 < W) {
            const float *row = L.I1 + (size_t)y * P;
            const float *up = L.I1 + (size_t)max(y - 1, 0) * P;
            const float *dn = L.I1 + (size_t)min(y + 1, H - 1) * P;
            float gx[4], gy[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int x = min(x0 + j, W - 1);
                gx[j] = 0.5f * (__ldg(row + min(x + 1, W - 1)) - __ldg(row + max(x - 1, 0)));
                gy[j] = 0.5f * (__ldg(dn + x) - __ldg(up + x));
            }
            st4(job.I1x + o, make_float4(gx[0], gx[1], gx[2], gx[3]));
            st4(job.I1y + o, make_float4(gy[0], gy[1], gy[2], gy[3]));
        }
    }
}

// A.2 "Warp (warpBackward)" for the whole level: reads u[cur], writes the four per-warp constants.
// The reference sums taps cx = ceil(wx-2) .. floor(wx+2) (4, or 5 when wx is integral, in which case
// both end taps have weight k(+-2) = 0).  Anchored at xmin = ceil(wx-2) the distance to tap xmin+4 is
// in [2,3), so its weight is always exactly 0: a fixed 4x4 window with separable weights gives the
// same sums (tap order preserved: rows outer, columns inner).
__device__ __forceinline__ void phase_warp(const int G, const int bid, const FusedJob &job, const FusedLevel &L, int cur) {
    const int W = L.w, H = L.h, P = L.pitch;
    const float *u1 = L.u1[cur], *u2 = L.u2[cur];
    const float *__restrict__ I1 = L.I1;
    const float *I1x = job.I1x, *I1y = job.I1y;  // written before the last grid barrier (which invalidated L1)
    // two pixels per thread and trip — the same column of two consecutive rows, so the two 6 x 6 tap windows share five rows in
    // L1 (the phase is latency-bound at 16 warps / SM: 64 independent gathers in flight per thread)
    const int hrows = (H + 1) >> 1;
    const int total = hrows * W;
    const int stride = G * kThreads;
    for (int i = bid * kThreads + threadIdx.x; i < total; i += stride) {
        const int yy = i / W, x = i - yy * W;
        const int y = 2 * yy;
        const bool has2 = y + 1 < H;
        const int y2 = has2 ? y + 1 : y, x2 = x;
        const size_t o = (size_t)y * P + x, o2 = (size_t)y2 * P + x2;
        float ix, iy, g, rc, jx, jy, g2, rc2;
        tvl1_warp_px_window(I1, I1x, I1y, W, H, P, x, y, u1[o], u2[o], __ldg(L.I0 + o), ix, iy, g, rc);
        tvl1_warp_px_window(I1, I1x, I1y, W, H, P, x2, y2, u1[o2], u2[o2], __ldg(L.I0 + o2), jx, jy, g2, rc2);
        job.I1wx[o] = ix;
        job.I1wy[o] = iy;
        job.grad[o] = tvl1_gq_from_grad(g);  // what the primal step wants of the gradient (tvl1_math.cuh)
        job.rho_c[o] = rc;
        if (has2) {
            job.I1wx[o2] = jx;
            job.I1wy[o2] = jy;
            job.grad[o2] = tvl1_gq_from_grad(g2);
            job.rho_c[o2] = rc2;
        }
    }
}

// A.2 step 4: upsample this level's flow to the next finer level (explicit dsize), x float(1/scaleStep)
__device__ __forceinline__ void phase_upsample(const int G, const int bid, const FusedJob &job, const FusedLevel &L, const FusedLevel &F, int cur) {
    const int total = F.h * F.w;
    for (int i = bid * kThreads + threadIdx.x; i < total; i += G * kThreads) {
        const int dy = i / F.w, dx = i - dy * F.w;
        const float sx = dx * L.up_fx, sy = dy * L.up_fy;
        const int x1 = __float2int_rd(sx), y1 = __float2int_rd(sy);
        const int x2 = x1 + 1, y2 = y1 + 1;
        const size_t r1 = (size_t)min(y1, L.h - 1) * L.pitch, r2 = (size_t)min(y2, L.h - 1) * L.pitch;
        const int x1r = min(x1, L.w - 1), x2r = min(x2, L.w - 1);
        const float w11 = (x2 - sx) * (y2 - sy), w12 = (sx - x1) * (y2 - sy);
        const float w21 = (x2 - sx) * (sy - y1), w22 = (sx - x1) * (sy - y1);
        const float *a = L.u1[cur], *b = L.u2[cur];
        float o1 = 0.f, o2 = 0.f;
        o1 = o1 + __ldcg(a + r1 + x1r) * w11;
        o1 = o1 + __ldcg(a + r1 + x2r) * w12;
        o1 = o1 + __ldcg(a + r2 + x1r) * w21;
        o1 = o1 + __ldcg(a + r2 + x2r) * w22;
        o2 = o2 + __ldcg(b + r1 + x1r) * w11;
        o2 = o2 + __ldcg(b + r1 + x2r) * w12;
        o2 = o2 + __ldcg(b + r2 + x1r) * w21;
        o2 = o2 + __ldcg(b + r2 + x2r) * w22;
        F.u1[0][(size_t)dy * F.pitch + dx] = o1 * job.up_mul;
        F.u2[0][(size_t)dy * F.pitch + dx] = o2 * job.up_mul;
    }
}

// A.5: merge(u1,u2) -> CV_32FC2
__device__ __forceinline__ void phase_merge(const int G, const int bid, const FusedJob &job, const FusedLevel &L, int cur) {
    const int total = L.h * L.w;
    if (job.bound > 0) {  // convertFlowToImage as the epilogue: 2 B/px leave the kernel instead of 8
        const double lo = -(double)job.bound, hi = (double)job.bound;
        for (int i = bid * kThreads + threadIdx.x; i < total; i += G * kThreads) {
            const int y = i / L.w, x = i - y * L.w;
            const size_t o = (size_t)y * L.pitch + x;
            job.qx[(size_t)y * job.q_pitch + x] = quantise_px(__ldcg(L.u1[cur] + o), lo, hi);
            job.qy[(size_t)y * job.q_pitch + x] = quantise_px(__ldcg(L.u2[cur] + o), lo, hi);
        }
        return;
    }
    for (int i = bid * kThreads + threadIdx.x; i < total; i += G * kThreads) {
        const int y = i / L.w, x = i - y * L.w;
        const size_t o = (size_t)y * L.pitch + x;
        float2 *row = reinterpret_cast<float2 *>(reinterpret_cast<char *>(job.flow_xy) + (size_t)y * job.flow_pitch_bytes);
        row[x] = make_float2(__ldcg(L.u1[cur] + o), __ldcg(L.u2[cur] + o));
    }
}

// ---- the register-tile inner loop -------------------------------------------------------------
// Tile (tx, ty) has its region origin at (tx*iw, ty*ih) (image coordinates, never negative), where
// iw = TW - 2hx, ih = TH - 2hy.  After kk <= min(hx, hy) iterations a pixel is valid unless it lies
// within the halo of a region edge that is NOT an image border: the first tile row/column keeps its
// top/left margin (the region edge is the image edge, where p(-1) = 0 is exactly the zero a region
// edge supplies), later tiles start their interior hx / hy in; the right/bottom margins are clipped
// by the image.  Reads state [cur], writes the interior to [cur^1].
//
// Warps synchronise only with their vertical neighbours, through progress counters in shared
// memory (sm.prog): warp q publishes row 0 of its new u after each primal step and row RPT-1 of its
// new p12/p22 after each dual step; the primal step of iteration i waits for warp q-1 to have
// finished dual(i-1), the dual step for warp q+1 to have finished primal(i).  Warps therefore drift
// apart by up to one half-step per row block, which overlaps the MUFU-heavy dual phase of some
// warps with the FMA-heavy primal phase of others, and no CTA-wide barrier sits in the loop.
// `base` is the counter value that means "tile loaded"; it advances by 2*kk + 2 per tile.
//
// Index-clamped forward differences (u(x+1) = u(x) on the last column / row): the pixel just outside
// the image is overwritten with a copy of the border pixel after every primal step, so the
// difference is exactly 0 without per-pixel masking; only tiles touching that border pay for it.
// Returns this thread's share of sum(diff) of the last primal step when `check`.
// Poll a neighbour warp's progress counter.  The loads are acquire loads: the (plain) loads of the neighbour's rows that
// follow must not be moved ahead of the poll — with a volatile poll ptxas hoisted the LDS.128 of the row below above the
// spin loop (seen in SASS), and results differed run to run.
__device__ __forceinline__ void wait_ge(const volatile int *flag, int v) {
    const unsigned addr = smem_u32(const_cast<const int *>(flag));
    int x;
    do {
        asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(x) : "r"(addr) : "memory");
    } while (x - v < 0);
}
__device__ __forceinline__ void signal(volatile int *flag, int v) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0)  // release store: this warp's rows (ordered before by __syncwarp) are visible before the counter
        asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"(smem_u32(const_cast<const int *>(flag))), "r"(v) : "memory");
}

// What one thread needs to know about the tile it is working on; everything here is loop-invariant over the kk
// iterations of a tile visit.
struct TileCtx {
    int so0;          // this thread's slot in row 0 of its warp in the shared-memory planes
    int lane, wq;
    int base;         // progress-counter value that means "tile loaded"
    bool flagsync;    // neighbour-warp progress counters (true) or CTA-wide barriers (false, debug / comparison)
    int jlast, rbot;  // EDGE tiles: pixel j == jlast of this lane is the last image column, row r == rbot of this warp the last image row
    bool edge_x, edge_y;
    bool lane_in;     // ERR: this lane's pixels lie in the interior columns of the tile
    int ry_lo, ry_hi, rows_left;  // ERR: interior rows of the tile, image rows below gy0
    int cols_left;    // ERR: image columns from gx0 (pixel j counts if j < cols_left)
};

// One primal + dual iteration of a tile visit.  EDGE: the tile contains the last image column or row (mirror handling
// for the index-clamped forward differences); ERR: accumulate this thread's share of sum(diff) of the primal step.
// Interior tiles in the middle of an epoch (the common case) instantiate neither.
//
// Order inside a warp (rows r = 0 .. RPT-1 of its block):   P0 | P1 D0 | P2 D1 | P3 D2 | D3
// The dual step of row r needs the new u of rows r and r+1 only, and the primal step of row r+1 needs the OLD p of row r,
// so D(r) can follow P(r+1) directly.  That puts the MUFU-bound dual arithmetic of one row next to the FMA-bound primal
// arithmetic of the next in one instruction stream (neighbouring warps are forced into near lock-step by their
// dependencies, so with "all primal, then all dual" every warp of the SM sat in the same phase and the two pipes took
// turns idling).  It also shortens the cross-warp chain: the warp above needs only this warp's P0 for its D3, and this
// warp's next P0 needs only the D3 of the warp above.
template <bool EDGE, bool ERR>
__device__ __forceinline__ void tile_iteration(Smem &sm, const TileCtx &t, const Tvl1Consts &c, int it, float4 (&p11)[RPT], float4 (&p12)[RPT],
                                               float4 (&p21)[RPT], float4 (&p22)[RPT], float &err) {
    volatile int *prog = sm.prog;
    const int so0 = t.so0, lane = t.lane, wq = t.wq;
    // p above the region's first row: the image border (p = 0) for tile row 0, halo garbage otherwise
    float4 up12 = zero4(), up22 = zero4();
    if (wq > 0) {
        if (t.flagsync) wait_ge(&prog[wq - 1], t.base + 2 * it);  // D3 of the previous iteration of the warp above
        up12 = *reinterpret_cast<const float4 *>(&sm.p_bot[0][wq - 1][4 * lane]);
        up22 = *reinterpret_cast<const float4 *>(&sm.p_bot[1][wq - 1][4 * lane]);
    }
    float4 c1 = zero4(), c2 = zero4();  // new u of the previous row (the dual step's centre row)
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
        // -------- primal, row r: u <- u + d(rho) + theta * div p ---------------------------------
        const int so = so0 + r * TW;
        const float4 ix = *reinterpret_cast<const float4 *>(&sm.consts[0][so]);
        const float4 iy = *reinterpret_cast<const float4 *>(&sm.consts[1][so]);
        const float4 gq = *reinterpret_cast<const float4 *>(&sm.consts[2][so]);
        const float4 rc = *reinterpret_cast<const float4 *>(&sm.consts[3][so]);
        const float4 o1 = *reinterpret_cast<const float4 *>(&sm.u[0][so]);
        const float4 o2 = *reinterpret_cast<const float4 *>(&sm.u[1][so]);
        float l11 = __shfl_up_sync(0xffffffffu, p11[r].w, 1);
        float l21 = __shfl_up_sync(0xffffffffu, p21[r].w, 1);
        if (lane == 0) l11 = l21 = 0.f;  // region edge: image border (p = 0) for tile column 0, halo otherwise
        float4 n1, n2;
        tvl1_primal_row(ix, iy, gq, rc, o1, o2, p11[r], l11, p12[r], r == 0 ? up12 : p12[r - 1], p21[r], l21, p22[r], r == 0 ? up22 : p22[r - 1], c, n1, n2);
        if (ERR) {
            const int ry = RPT * wq + r;
            if (t.lane_in && ry >= t.ry_lo && ry < t.ry_hi && r < t.rows_left) {
                const float4 d = tvl1_diff_row(o1, o2, n1, n2);
                err += d.x;
                if (1 < t.cols_left) err += d.y;
                if (2 < t.cols_left) err += d.z;
                if (3 < t.cols_left) err += d.w;
            }
        }
        if (EDGE) {
            if (t.edge_x) {  // mirror the last image column into the pixel right of it: u(x+1) - u(x) == 0 there
                if (t.jlast == 0) { n1.y = n1.x; n2.y = n2.x; }
                if (t.jlast == 1) { n1.z = n1.y; n2.z = n2.y; }
                if (t.jlast == 2) { n1.w = n1.z; n2.w = n2.z; }
            }
            if (t.edge_y && r > 0 && r - 1 == t.rbot) {  // first out-of-image row: a copy of the last image row
                n1 = c1;
                n2 = c2;
            }
        }
        st4(&sm.u[0][so], n1);
        st4(&sm.u[1][so], n2);
        if (r == 0) {
            signal(&prog[wq], t.base + 2 * it + 1);  // row 0 of the new u is what the warp above waits for
            if (!t.flagsync) __syncthreads();
        } else {
            // -------- dual, row r-1: p <- (p + taut * grad u) / (1 + taut * |grad u|) ------------
            float r1 = __shfl_down_sync(0xffffffffu, c1.x, 1);
            float r2 = __shfl_down_sync(0xffffffffu, c2.x, 1);
            if (EDGE && t.edge_x && t.jlast == 3) {
                r1 = c1.w;
                r2 = c2.w;
            }
            tvl1_dual_row(c1, c2, n1, n2, r1, r2, c.taut, p11[r - 1], p12[r - 1], p21[r - 1], p22[r - 1]);
        }
        c1 = n1;
        c2 = n2;
    }
    // -------- dual, last row: the row below belongs to the next warp (its P0 of this iteration) ----
    {
        float4 d1 = c1, d2 = c2;  // region's last row: halo, or the mirrored image border
        if (wq < kWarps - 1) {
            if (t.flagsync) wait_ge(&prog[wq + 1], t.base + 2 * it + 1);
            if (!(EDGE && t.edge_y && t.rbot == RPT - 1)) {
                d1 = *reinterpret_cast<const float4 *>(&sm.u[0][so0 + RPT * TW]);
                d2 = *reinterpret_cast<const float4 *>(&sm.u[1][so0 + RPT * TW]);
            }
        }
        float r1 = __shfl_down_sync(0xffffffffu, c1.x, 1);
        float r2 = __shfl_down_sync(0xffffffffu, c2.x, 1);
        if (EDGE && t.edge_x && t.jlast == 3) {
            r1 = c1.w;
            r2 = c2.w;
        }
        tvl1_dual_row(c1, c2, d1, d2, r1, r2, c.taut, p11[RPT - 1], p12[RPT - 1], p21[RPT - 1], p22[RPT - 1]);
    }
    st4(&sm.p_bot[0][wq][4 * lane], p12[RPT - 1]);
    st4(&sm.p_bot[1][wq][4 * lane], p22[RPT - 1]);
    signal(&prog[wq], t.base + 2 * it + 2);
    if (!t.flagsync) __syncthreads();
}

template <bool EDGE>
__device__ __forceinline__ float tile_iterations(Smem &sm, const TileCtx &t, const Tvl1Consts &c, int kk, bool check, float4 (&p11)[RPT],
                                                 float4 (&p12)[RPT], float4 (&p21)[RPT], float4 (&p22)[RPT]) {
    float err = 0.f;
    const int plain = check ? kk - 1 : kk;
    for (int it = 0; it < plain; ++it) tile_iteration<EDGE, false>(sm, t, c, it, p11, p12, p21, p22, err);
    if (check) tile_iteration<EDGE, true>(sm, t, c, kk - 1, p11, p12, p21, p22, err);
    return err;
}

__device__ __forceinline__ float process_tile(const FusedJob &job, const Tvl1Consts &c, const FusedLevel &L, int level, int cur, int tx, int ty,
                                              int kk, int hx, int hy, bool check, int base, unsigned tma_parity, Smem &sm,
                                              bool prof_on, int ntx_next, int nty_next) {
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    unsigned long long t0 = 0;
    if (prof_on) t0 = gtime();
    const int W = L.w, H = L.h, P = L.pitch;
    const int rx0 = tx * (TW - 2 * hx), ry0 = ty * (TH - 2 * hy);
    const int gx0 = rx0 + 4 * lane;
    const int gy0 = ry0 + RPT * wq;
    volatile int *prog = sm.prog;
    const bool flagsync = job.flag_sync != 0;

    float4 p11[RPT], p12[RPT], p21[RPT], p22[RPT];
    const int so0 = (RPT * wq) * TW + 4 * lane;  // this thread's slot in row 0 of its warp (thread-private in smem planes)
    const bool use_tma = job.use_tma != 0;
    if (use_tma) {
        // One thread stages the six shared-memory-resident planes of the tile (4 constants + u1,u2: 192 KB) with
        // TMA while every thread loads its share of the four dual planes into registers.  All warps must be done
        // with the previous tile's shared memory first (the bulk copy overwrites every slot).
        fence_proxy_async();
        __syncthreads();
        if (threadIdx.x == 0) {
            const char *maps = static_cast<const char *>(job.tmaps) + (size_t)level * kFusedMapsPerLevel * kTensorMapBytes;
            // the planes were written with plain stores by other CTAs of the lane (previous chunk / warp phase) and published by
            // the grid barrier this thread polled: order those generic-proxy writes before the async-proxy reads below
            fence_proxy_async_global();
            mbar_expect_tx(&sm.tma_bar, 6u * kConstPlane * (unsigned)sizeof(float));
            tma_load_2d(sm.consts[0], maps + 0 * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
            tma_load_2d(sm.consts[1], maps + 1 * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
            tma_load_2d(sm.consts[2], maps + 2 * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
            tma_load_2d(sm.consts[3], maps + 3 * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
            tma_load_2d(sm.u[0], maps + (4 + 2 * cur) * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
            tma_load_2d(sm.u[1], maps + (5 + 2 * cur) * kTensorMapBytes, rx0, ry0, &sm.tma_bar);
        }
    } else if (flagsync && wq > 0) {
        // The warp above reads this warp's first u row in its dual steps: it must have finished the previous tile
        // (its counter reached base - 2 = "last dual step of the previous tile done") before the row is overwritten.
        wait_ge(&prog[wq - 1], base - 2);
    }
    {
        const float *s0 = L.u1[cur], *s1 = L.u2[cur], *s2 = job.p[cur][0], *s3 = job.p[cur][1], *s4 = job.p[cur][2],
                    *s5 = job.p[cur][3];
        const bool col_ok = gx0 < P;
#pragma unroll
        for (int r = 0; r < RPT; ++r) {
            const int gy = gy0 + r;
            const bool ok = col_ok && gy < H;
            const size_t o = ok ? (size_t)gy * P + gx0 : 0;
            p11[r] = ok ? ld_cg4(s2 + o) : zero4();
            p12[r] = ok ? ld_cg4(s3 + o) : zero4();
            p21[r] = ok ? ld_cg4(s4 + o) : zero4();
            p22[r] = ok ? ld_cg4(s5 + o) : zero4();
            if (!use_tma) {
                const int so = so0 + r * TW;
                st4(&sm.u[0][so], ok ? ld_cg4(s0 + o) : zero4());
                st4(&sm.u[1][so], ok ? ld_cg4(s1 + o) : zero4());
                st4(&sm.consts[0][so], ok ? ld_cg4(job.I1wx + o) : zero4());
                st4(&sm.consts[1][so], ok ? ld_cg4(job.I1wy + o) : zero4());
                st4(&sm.consts[2][so], ok ? ld_cg4(job.grad + o) : zero4());
                st4(&sm.consts[3][so], ok ? ld_cg4(job.rho_c + o) : zero4());
            }
        }
    }
    if (use_tma) mbar_wait(&sm.tma_bar, tma_parity);
    if (job.prefetch && ntx_next >= 0) {
        // This CTA's next tile of the chunk: ask for its ten planes to be brought into L2 now, so the copy from HBM runs
        // under this tile's iterations (with several pairs in flight the planes of a level do not fit the L2).
        const int nrx0 = ntx_next * (TW - 2 * hx), nry0 = nty_next * (TH - 2 * hy);
        if (use_tma && threadIdx.x == 0) {
            const char *maps = static_cast<const char *>(job.tmaps) + (size_t)level * kFusedMapsPerLevel * kTensorMapBytes;
            tma_prefetch_l2_2d(maps + 0 * kTensorMapBytes, nrx0, nry0);
            tma_prefetch_l2_2d(maps + 1 * kTensorMapBytes, nrx0, nry0);
            tma_prefetch_l2_2d(maps + 2 * kTensorMapBytes, nrx0, nry0);
            tma_prefetch_l2_2d(maps + 3 * kTensorMapBytes, nrx0, nry0);
            tma_prefetch_l2_2d(maps + (4 + 2 * cur) * kTensorMapBytes, nrx0, nry0);
            tma_prefetch_l2_2d(maps + (5 + 2 * cur) * kTensorMapBytes, nrx0, nry0);
        }
        if ((lane & 7) == 0) {  // one lane per 128-byte line of the four dual planes
            const int ngx = nrx0 + 4 * lane;
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const int ngy = nry0 + RPT * wq + r;
                if (ngx < P && ngy < H) {
                    const size_t o = (size_t)ngy * P + ngx;
                    prefetch_l2(job.p[cur][0] + o);
                    prefetch_l2(job.p[cur][1] + o);
                    prefetch_l2(job.p[cur][2] + o);
                    prefetch_l2(job.p[cur][3] + o);
                }
            }
        }
    }
    TileCtx t;
    t.so0 = so0;
    t.lane = lane;
    t.wq = wq;
    t.base = base;
    t.flagsync = flagsync;
    // image borders inside this tile's region (tile-uniform)
    t.edge_x = W - 1 >= rx0 && W - 1 < rx0 + TW;
    t.edge_y = H - 1 >= ry0 && H - 1 < ry0 + TH;
    t.jlast = W - 1 - gx0;
    t.rbot = H - 1 - gy0;
    // which of this thread's pixels are interior (written back / counted in the error)
    t.lane_in = (tx == 0 || 4 * lane >= hx) && 4 * lane < TW - hx + (rx0 + TW >= W ? hx : 0) && gx0 < W;
    t.ry_lo = ty == 0 ? 0 : hy;
    t.ry_hi = TH - hy + (ry0 + TH >= H ? hy : 0);
    t.rows_left = H - gy0;
    t.cols_left = W - gx0;

    // make row RPT-1 of p12/p22 visible to the warp below before the first primal step
    st4(&sm.p_bot[0][wq][4 * lane], p12[RPT - 1]);
    st4(&sm.p_bot[1][wq][4 * lane], p22[RPT - 1]);
    signal(&prog[wq], base);
    if (!flagsync) __syncthreads();
    if (prof_on) {
        const unsigned long long tt = gtime();
        sm.prof[5] += tt - t0;
        t0 = tt;
    }

    const float err = (t.edge_x || t.edge_y) ? tile_iterations<true>(sm, t, c, kk, check, p11, p12, p21, p22)
                                             : tile_iterations<false>(sm, t, c, kk, check, p11, p12, p21, p22);
    if (prof_on) {
        const unsigned long long tt = gtime();
        sm.prof[6] += tt - t0;
        t0 = tt;
    }
    // -------- write the interior to the other buffer ---------------------------------------------
    {
        float *d0 = L.u1[cur ^ 1], *d1 = L.u2[cur ^ 1], *d2 = job.p[cur ^ 1][0], *d3 = job.p[cur ^ 1][1],
              *d4 = job.p[cur ^ 1][2], *d5 = job.p[cur ^ 1][3];
#pragma unroll
        for (int r = 0; r < RPT; ++r) {
            const int ry = RPT * wq + r, gy = gy0 + r;
            if (t.lane_in && ry >= t.ry_lo && ry < t.ry_hi && gy < H) {
                const size_t o = (size_t)gy * P + gx0;
                st4(d0 + o, *reinterpret_cast<const float4 *>(&sm.u[0][so0 + r * TW]));
                st4(d1 + o, *reinterpret_cast<const float4 *>(&sm.u[1][so0 + r * TW]));
                st4(d2 + o, p11[r]);
                st4(d3 + o, p12[r]);
                st4(d4 + o, p21[r]);
                st4(d5 + o, p22[r]);
            }
        }
    }
    if (prof_on) sm.prof[7] += gtime() - t0;
    return err;
}

// tiles needed along one axis: tile i covers up to i*(T-2h) + T (clipped by the image) minus a halo that
// only matters when the image continues beyond the region
__host__ __device__ __forceinline__ int tiles_along(int n, int T, int h) { return fused_tiles_along(n, T, h); }

// phase profiler (CTA 0 / thread 0 only): attributes wall time between marks to a category
struct Prof {
    unsigned long long *acc;  // shared memory
    unsigned long long last;
    bool on;
    __device__ void init(unsigned long long *a, bool first_cta) {
        acc = a;
        on = first_cta && threadIdx.x == 0;
        if (on) {
            for (int i = 0; i < 32; ++i) acc[i] = 0;
            last = gtime();
        }
    }
    __device__ __forceinline__ void mark(int cat, int cat2 = -1) {
        if (on) {
            const unsigned long long t = gtime();
            acc[cat] += t - last;
            if (cat2 >= 0) acc[cat2] += t - last;
            last = t;
        }
    }
};

// where a CTA finds its lane's job: the parameter bank (<= 16 lanes), or a copy in shared memory of the device-memory ring entry
__device__ __forceinline__ const FusedJob &job_of(const FusedBatchParams &batch, int lane_id, Smem &) { return batch.job[lane_id]; }
__device__ __forceinline__ const FusedJob &job_of(const FusedBatch &batch, int lane_id, Smem &sm) {
    const int *src = reinterpret_cast<const int *>(batch.jobs + lane_id);
    int *dst = reinterpret_cast<int *>(&sm.job);
    for (int i = threadIdx.x; i < (int)(sizeof(FusedJob) / sizeof(int)); i += kThreads) dst[i] = __ldg(src + i);
    __syncthreads();
    return sm.job;
}

template <class Batch>
__global__ void __launch_bounds__(kThreads, kFusedCtasPerSm) k_tvl1_pair(const __grid_constant__ Batch batch) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
    const int G = batch.group;
    const int lane_id = blockIdx.x / G, bid = blockIdx.x - lane_id * G;
    const FusedJob &job = job_of(batch, lane_id, sm);
    const Tvl1Consts c = job.c;  // by value: the job is indexed dynamically in the parameter bank
    unsigned epoch = 0;
    unsigned *bar = job.sync;
    int cur = 0;
    unsigned long long px_iters = 0, px_chunks = 0;
    int tile_base = 1;  // progress-counter epoch of the tile loop (sm.prog starts at 0)
    // convergence partials are double-buffered: a CTA that leaves the barrier early may already write the NEXT check's partial
    // while a slower one still sums this check's (at the small levels a 2-iteration chunk is a few microseconds); a divergent
    // sum would desynchronise the barrier counts.  One barrier of lead is the most any CTA can have, so two sets suffice.
    int part_sel = 0;
    unsigned tma_parity = 0;
    Prof prof;
    prof.init(sm.prof, bid == 0);
    if (threadIdx.x < kWarps) {
        sm.prog[threadIdx.x] = 0;
        sm.red[threadIdx.x] = 0.0;
    }
    if (threadIdx.x == 0) mbar_init(&sm.tma_bar, 1);
    __syncthreads();

    for (int s = job.nscales - 1; s >= 0; --s) {
        const FusedLevel &L = job.lv[s];
        cur = 0;  // level start: u[0] holds the upsampled (or zero) flow, p[0] is zeroed
        phase_level_start(G, bid, job, L, s == job.nscales - 1);
        prof.mark(0);
        grid_barrier(bar, epoch, G, job.ctl);
        prof.mark(3);
        const double scaled_eps = job.epsilon * job.epsilon * (double)((long long)L.w * L.h);  // A.4
        for (int wi = 0; wi < job.warps; ++wi) {
            phase_warp(G, bid, job, L, cur);
            prof.mark(1);
            grid_barrier(bar, epoch, G, job.ctl);
            prof.mark(3);
            double error = DBL_MAX, prev_error = 0.0;
            int n = 0;
            while (error > scaled_eps && n < job.iterations) {
                // plan the epoch: iterations up to and including the next convergence check (A.4)
                int K = 0, nn = n;
                bool check = false;
                double pp = prev_error;
                for (;;) {
                    const bool calc = job.epsilon > 0 && (nn & 1) && pp < scaled_eps;
                    ++K;
                    ++nn;
                    if (calc) {
                        check = true;
                        break;
                    }
                    pp -= scaled_eps;
                    if (nn >= job.iterations) break;
                }
                int remaining = K;
                while (remaining > 0) {
                    const int nch = (remaining + job.k - 1) / job.k;
                    const int kk = (remaining + nch - 1) / nch;
                    const bool chk = check && kk == remaining;
                    const int hx = (kk + 3) & ~3, hy = kk;
                    const int ntx = tiles_along(L.w, TW, hx), nty = tiles_along(L.h, TH, hy);
                    const int ntiles = ntx * nty;
                    for (int t = bid; t < ntiles; t += G) {
                        const int ty = t / ntx, tx = t - ty * ntx;
                        const int tn = t + G;
                        const int nty_n = tn < ntiles ? tn / ntx : -1, ntx_n = tn < ntiles ? tn - nty_n * ntx : -1;
                        const float e = process_tile(job, c, L, s, cur, tx, ty, kk, hx, hy, chk, tile_base, tma_parity, sm, prof.on, ntx_n, nty_n);
                        tile_base += 2 * kk + 2;
                        tma_parity ^= 1u;
                        if (chk) {  // per-warp running sums in shared memory: no CTA-wide barrier per tile
                            double v = (double)e;
#pragma unroll
                            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                            if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] += v;
                        }
                    }
                    if (chk) {  // one barrier per checking chunk: thread 0 adds the 16 warp sums in a fixed order
                        __syncthreads();
                        if (threadIdx.x == 0) {
                            double bs = 0.0;
#pragma unroll
                            for (int k = 0; k < kWarps; ++k) {
                                bs += sm.red[k];
                                sm.red[k] = 0.0;
                            }
                            job.partials[part_sel * kPartialSet + bid] = bs;
                        }
                    }
                    prof.mark(2, 8 + s);
                    if (prof.on) prof.acc[16 + s] += 1;
                    px_chunks += (unsigned long long)(L.w * L.h);
                    grid_barrier(bar, epoch, G, job.ctl);
                    prof.mark(3);
                    cur ^= 1;
                    remaining -= kk;
                }
                n = nn;
                if (check) {
                    // every CTA sums all partials in the same fixed order -> identical decisions everywhere
                    if (threadIdx.x < 32) {
                        double v = 0.0;
                        for (int i = threadIdx.x; i < G; i += 32) v += __ldcg(job.partials + part_sel * kPartialSet + i);
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                        if (threadIdx.x == 0) sm.bcast[0] = v;
                    }
                    __syncthreads();
                    error = sm.bcast[0];
                    __syncthreads();
                    part_sel ^= 1;
                    prev_error = error;
                } else {
                    error = DBL_MAX;
                    prev_error = pp;
                }
            }
            if (bid == 0 && threadIdx.x == 0) job.iters_log[s * job.warps + wi] = n;
            px_iters += (unsigned long long)n * (unsigned long long)(L.w * L.h);
        }
        if (s > 0) {
            phase_upsample(G, bid, job, L, job.lv[s - 1], cur);
            prof.mark(4);
            grid_barrier(bar, epoch, G, job.ctl);
            prof.mark(3);
        }
    }
    phase_merge(G, bid, job, job.lv[0], cur);
    prof.mark(4);
    if (prof.on)
        for (int i = 0; i < 32; ++i) job.ctl->prof[i] = prof.acc[i];
    if (bid == 0 && threadIdx.x == 0) {
        job.ctl->px_iters_total += px_iters;
        job.ctl->px_chunks_total += px_chunks;
    }  // single writer, launches are serialised

    // last CTA out resets the barrier words for the next launch
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned done = atomicAdd(bar + 1, 1u);
        if (done == (unsigned)G - 1) {
            bar[0] = 0;
            bar[1] = 0;
            __threadfence();
        }
    }
}

}  // namespace

void fused_encode_tensor_map(void *out, const float *plane, int w, int h, int pitch) {
    encode_tensor_map_2d(out, plane, w, h, pitch, TW, TH);
}

int fused_num_sms(int device) {
    static std::mutex m;
    static int num_sms[64] = {};
    if (device < 0 || device >= 64) return 132;
    std::lock_guard<std::mutex> lk(m);  // handles are created and used from several host threads (list workers)
    if (num_sms[device] == 0) DFB_CUDA(cudaDeviceGetAttribute(&num_sms[device], cudaDevAttrMultiProcessorCount, device));
    return num_sms[device];
}

template <class Batch>
static void configure_kernel() {
    DFB_CUDA(cudaFuncSetAttribute(k_tvl1_pair<Batch>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)));
    DFB_CUDA(cudaFuncSetAttribute(k_tvl1_pair<Batch>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int resident = 0;
    DFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, k_tvl1_pair<Batch>, kThreads, sizeof(Smem)));
    if (resident < kFusedCtasPerSm)
        throw std::runtime_error("k_tvl1_pair: only " + std::to_string(resident) + " CTA(s) fit an SM, the launch geometry needs " +
                                 std::to_string(kFusedCtasPerSm));
}

int launch_tvl1_fused(const FusedBatch &batch, int device, cudaStream_t s, bool serialise) {
    // the opt-in shared-memory size is a per-device function attribute: handles on several devices may live in one process
    static std::mutex mtx;
    static bool configured[64] = {};
    {
        std::lock_guard<std::mutex> lk(mtx);
        const int d = device >= 0 && device < 64 ? device : 0;
        if (!configured[d]) {
            configure_kernel<FusedBatch>();
            configure_kernel<FusedBatchParams>();
            configured[d] = true;
        }
    }
    static_assert(TW == kFusedTileW && TH == kFusedTileH, "tile geometry is shared with the host heuristics");
    // all CTAs must be co-resident: group * njobs <= SM count x kFusedCtasPerSm, enforced by the cooperative launch
    const int grid = batch.group * batch.njobs;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = sizeof(Smem);
    cfg.stream = s;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeCooperative;
    attrs[0].val.cooperative = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 1;
    // Two handles on one GPU (two list workers) launch this kernel from different streams.  Barriers are PER LANE, so a lane
    // of the second grid runs as soon as its own CTAs are resident: the second grid fills the SMs the first one's finished
    // lanes leave behind (+3.8 % on the 340x256 list, 4020 vs 3873 pairs/s).  The block scheduler hands out a later grid's
    // CTAs only after every CTA of the earlier grid has been placed, so an earlier grid is never starved by a later one; a
    // lost arrival would still surface through the barrier watchdog rather than hang.  `serialise` (engine knob
    // serial_launches) chains the launches of one device through an event for callers that want strict one-at-a-time
    // execution.
    {
        std::lock_guard<std::mutex> lk(mtx);
        const int d = device >= 0 && device < 64 ? device : 0;
        static cudaEvent_t last_done[64] = {};
        if (serialise) {
            if (!last_done[d]) DFB_CUDA(cudaEventCreateWithFlags(&last_done[d], cudaEventDisableTiming));
            else DFB_CUDA(cudaStreamWaitEvent(s, last_done[d], 0));
        }
        if (batch.njobs <= kFusedParamLanes) {
            FusedBatchParams pb;
            pb.njobs = batch.njobs;
            pb.group = batch.group;
            std::memcpy(pb.job, batch.host_jobs, sizeof(FusedJob) * batch.njobs);
            DFB_CUDA(cudaLaunchKernelEx(&cfg, k_tvl1_pair<FusedBatchParams>, pb));
        } else {
            DFB_CUDA(cudaLaunchKernelEx(&cfg, k_tvl1_pair<FusedBatch>, batch));
        }
        if (serialise) DFB_CUDA(cudaEventRecord(last_done[d], s));
    }
    return 1;
}

}  // namespace dfb
