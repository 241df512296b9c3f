// tvl1_fused.cuh — the persistent fused TV-L1 pair kernel (tvl1_fused.cu): job description shared
// between the host engine and the device code.
#pragma once

#include "tma.cuh"
#include "tvl1.cuh"

namespace dfb {

constexpr int kFusedMaxK = 8;  // most inner iterations kept on chip per tile visit (halo width)

struct FusedLevel {
    int w, h, pitch;
    const float *I0, *I1;  // pyramid level of frame a / frame b
    float *u1[2], *u2[2];  // flow, ping-pong
    float up_fx, up_fy;    // resize factors for upsampling THIS level's flow to level-1 (A.2 step 4)
};

// Written by the kernel into mapped host memory (no memcpy, no sync on the pair path).
struct FusedHostCtl {
    double error;         // unfused engine: convergence sum read by the host state machine
    unsigned long long px_iters_total;  // sum over pairs of (level pixels x executed iterations)
    unsigned long long px_chunks_total; // sum over pairs of (level pixels x tile visits): 64 B of state/constant traffic each
    // CTA-0 view of where the last pair's time went, in ns (globaltimer): [0] level start, [1] warps,
    // [2] tile compute, [3] grid barriers, [4] upsample+merge, [8+s] tile compute at scale s, [16+s] chunks at scale s,
    // [24] median filtering
    unsigned long long prof[32];
    // watchdog of the grid barrier: a CTA that polls the arrival counter kFusedStallPolls times (an L2 round trip each: 10-25 s)
    // records {1, blockIdx.x, barrier target, counter value, CTAs per lane, lane} here and traps, so a lost arrival surfaces
    // as a CUDA error instead of a hung device
    unsigned stall[8];
};
constexpr unsigned kFusedStallPolls = 1u << 25;

struct FusedJob {
    int nscales, warps, iterations, k;
    int use_tma;    // 1: constants + u tiles staged by TMA (cp.async.bulk.tensor.2d), 0: LDG -> STS
    int median_k;   // 3 or 5: u1, u2 <- their k x k median before every iteration n of a warp with n % median_interval == 0; 0: off
    // CUtensorMap[nscales][kFusedMapsPerLevel] in global memory: I1wx, I1wy, grad, rho_c, u1[0], u2[0], u1[1], u2[1]
    const void *tmaps;
    double epsilon;
    Tvl1Consts c;
    float up_mul;
    FusedLevel lv[16];
    float *I1x, *I1y, *I1wx, *I1wy, *grad, *rho_c;
    float *p[2][4];  // p11,p12,p21,p22 ping-pong
    double *partials;
    unsigned *sync;
    FusedHostCtl *ctl;
    int *iters_log;  // [16 * 16] executed inner iterations per (scale, warp) of THIS pair, index s * warps + w (mapped host memory)
    float *flow_xy;
    size_t flow_pitch_bytes;
    // bound > 0: emit the two quantised uint8 planes instead of the float2 field (PairJob)
    int bound;
    int median_interval;  // see median_k
    int init_flow;  // 1: the coarsest level starts from the flow already in its u1[0] / u2[0] (use_initial_flow) instead of 0
    uint8_t *qx, *qy;
    size_t q_pitch;
    // fx non-null: emit u1 / u2 as two float planes instead of the float2 field (PairJob)
    float *fx, *fy;
    size_t f_pitch;
};

// Several independent pairs ("lanes") per launch: lane i is solved by CTAs [i*group, (i+1)*group) with
// their own barrier words, partials and workspace.  Coarse pyramid levels have fewer tiles than the
// GPU has SMs; running pairs side by side keeps every SM busy without touching a pair's arithmetic.
constexpr int kFusedMaxLanes = 64;  // job descriptions travel through a device-memory ring, not the parameter bank
constexpr int kFusedMapsPerLevel = 8;
constexpr int kFusedParamLanes = 16;  // 16 jobs x 1.4 KB fit the kernel parameter bank (32 KB)
struct FusedBatch {
    int njobs, group;
    const FusedJob *jobs;  // njobs > kFusedParamLanes: [njobs] in device memory, each CTA copies its lane's job into shared memory
    const FusedJob *host_jobs;  // the same descriptions in host memory (always); copied into the parameter bank when they fit
};
// njobs <= kFusedParamLanes: the jobs travel in the parameter bank (uniform loads, no registers or shared memory spent on them —
// 4 % faster at 1080p than reading them from shared memory)
struct FusedBatchParams {
    int njobs, group;
    FusedJob job[kFusedParamLanes];
};

// tiles needed along one axis (see process_tile): region origins at multiples of T - 2h
__host__ __device__ inline int fused_tiles_along(int n, int T, int h) {
    const int stride = T - 2 * h;
    return n <= T ? 1 : (n - 2 * h + stride - 1) / stride;
}
constexpr int kFusedTileW = 128, kFusedTileH = 64;
// CTAs of the persistent kernel resident per SM: a 512-thread CTA owns the whole SM (192 KB tile)
constexpr int kFusedCtasPerSm = 1;
constexpr int kFusedDefaultK = 8;

int fused_num_sms(int device);
inline int fused_cta_slots(int device) { return fused_num_sms(device) * kFusedCtasPerSm; }
// Encodes one 2-D fp32 descriptor of one warp's rows of a tile (box 128 x 4, no swizzle, zero fill out of bounds)
// into out[128 bytes].
// plane: base pointer, extent w x h (elements / rows), row pitch in elements.
void fused_encode_tensor_map(void *out, const float *plane, int w, int h, int pitch);
// gamma > 0 (SURVEY A.8): lane i's illumination field (u3[l]: level l of its pyramid) and dual planes p31, p32.  Passed beside
// the jobs rather than in FusedJob, so k_tvl1_pair's job layout and code do not change.
struct FusedGammaLane {
    float *u3[16];
    float *p31, *p32;
};
struct FusedGamma {
    float gamma;
    FusedGammaLane lane[kFusedMaxLanes];
};
// returns the number of kernels launched; gm non-null (gamma > 0): the gamma kernel k_tvl1_pair_gamma (DESIGN §4.3)
int launch_tvl1_fused(const FusedBatch &batch, int device, cudaStream_t s, const FusedGamma *gm = nullptr);

// Test hook: one phase of k_tvl1_pair (its own device functions) on up to kFusedParamLanes lanes in one cooperative launch.
enum FusedStage : int {
    kFusedStageLevelStart,  // phase_level_start at level `level` (coarsest: zero u too, unless the job's init_flow is set)
    kFusedStageWarp,        // phase_warp at level `level` from u[0]
    kFusedStageGq,          // grad -> tvl1_gq_from_grad(grad) over the level's plane
    kFusedStageChunks,      // n chunks of kk iterations at level `level` from state [0], every one checking when `check`
    kFusedStageUpsample,    // phase_upsample from level `level` (u[0]) to level `level` - 1
    kFusedStageMerge,       // phase_merge of level `level` (u[0])
    kFusedStageMedian,      // phase_median of level `level` with window kk, u[0] -> u[1]
};
struct FusedStageArgs {
    int stage, level, coarsest, kk, n, check;
};
void launch_tvl1_stage(const FusedBatch &batch, const FusedStageArgs &a, cudaStream_t s);

}  // namespace dfb
