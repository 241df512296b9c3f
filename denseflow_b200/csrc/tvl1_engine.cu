// tvl1_engine.cu — host orchestration of the TV-L1 path: the replacement for
// cv::cuda::OpticalFlowDual_TVL1 as created/called at /root/reference/src/denseflow_gpu.cpp:299,327
// (control flow per SURVEY.md Appendix A.1, A.2, A.4, A.5).
//
// Two schedules over the same arithmetic:
//   fused = 1 (default)  one persistent cooperative kernel per pair (tvl1_fused.cu): gradients,
//                        warps, the primal/dual iterations with k steps kept on chip per tile, the
//                        A.4 convergence state machine and the flow upsampling all run on-device
//                        with no host round trip.
//   fused = 0            one kernel per half-step, the reference's launch structure, with the A.4
//                        state machine on the host (one stream sync per convergence check).
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "engine.h"
#include "tvl1.cuh"
#include "tvl1_fused.cuh"

namespace dfb {

namespace {

constexpr int kMaxScales = 16;
constexpr int kMaxWarps = 16;  // the iteration log holds kMaxScales x kMaxWarps entries per pair
constexpr double kAllocScaleStep = 0.8;  // scaleStep the slot / lane pyramid layout is sized for (the create() default)

struct Tvl1Params {
    double tau = 0.25, lambda = 0.15, theta = 0.3;
    int nscales = 5, warps = 5;
    double epsilon = 0.01;
    int iterations = 300;
    double scale_step = 0.8;
    int fused = 1;
    int fused_k = kFusedDefaultK;
    int time_kernels = 0;
    int use_tma = 1;
    int lanes = 0;  // pairs solved side by side per fused launch; 0 = choose from the tile counts
    int median_filtering = 0;  // 3 or 5: the window of the median of u1, u2 between iterations (DESIGN §4.3); 0 or 1: off
    int median_interval = 30;  // the median runs before every iteration n of a warp with n % median_interval == 0
    int use_initial_flow = 0;  // 1: each pair starts from the flow its call passes in (PairJob::init_x; DESIGN §1)
    double gamma = 0;  // > 0: weight of the illumination field u3 (SURVEY A.8; DESIGN §4.3)
    int median_k() const { return median_filtering > 1 ? median_filtering : 0; }
};

class Tvl1 final : public FlowAlgorithm {
  public:
    Tvl1(int device, int max_w, int max_h) : device_(device), max_w_(max_w), max_h_(max_h) {
        DFB_CUDA(cudaSetDevice(device_));
        allocate();
    }
    ~Tvl1() override {
        cudaSetDevice(device_);
        for (auto &l : lanes_) {
            if (l.host_ctl) cudaFreeHost(l.host_ctl);
            if (l.own) cudaFree(l.own);
            if (l.tmaps) cudaFree(l.tmaps);
        }
        if (stats_event_) cudaEventDestroy(stats_event_);
        if (pair_log_) cudaFreeHost(pair_log_);
        if (unfused_scratch_) cudaFree(unfused_scratch_);
        for (auto &l : lanes_)
            if (l.gamma_own) cudaFree(l.gamma_own);
        for (int r = 0; r < kJobRing; ++r) {
            if (job_ring_h_[r]) cudaFreeHost(job_ring_h_[r]);
            if (job_ring_d_[r]) cudaFree(job_ring_d_[r]);
            if (job_ring_ev_[r]) cudaEventDestroy(job_ring_ev_[r]);
        }
    }
    const char *name() const override { return "tvl1"; }

    // A refused value leaves the parameter as it was.  tau and theta must be positive: the dual step's 1 + taut * |grad u|
    // >= 1 and the primal clamp's l_t >= 0 rely on it (tvl1_math.cuh).
    bool set_param(const std::string &k, double v) override {
        if (k == "tau") { if (!(std::isfinite(v) && v > 0)) return false; prm_.tau = v; }
        else if (k == "lambda") { if (!(std::isfinite(v) && v >= 0)) return false; prm_.lambda = v; }
        else if (k == "theta") { if (!(std::isfinite(v) && v > 0)) return false; prm_.theta = v; }
        else if (k == "nscales") { if (!whole_in(v, 1, kMaxScales)) return false; prm_.nscales = (int)v; }
        else if (k == "warps") { if (!whole_in(v, 1, kMaxWarps)) return false; prm_.warps = (int)v; }
        else if (k == "epsilon") { if (!std::isfinite(v)) return false; prm_.epsilon = v; }  // <= 0: no convergence checks
        else if (k == "iterations") { if (!whole_in(v, 1, INT_MAX)) return false; prm_.iterations = (int)v; }
        else if (k == "scale_step") {
            // the pyramid slots were laid out at create time for the default 0.8: a larger factor would not fit them
            if (!(v > 0 && v <= kAllocScaleStep)) return false;
            prm_.scale_step = v;
        }
        else if (k == "fused") { if (!is_flag(v)) return false; prm_.fused = (int)v; }
        else if (k == "fused_k") { if (!whole_in(v, 1, kFusedMaxK) || 2 * v >= kFusedTileH) return false; prm_.fused_k = (int)v; }
        else if (k == "time_kernels") { if (!is_flag(v)) return false; prm_.time_kernels = (int)v; }
        else if (k == "use_tma") { if (!is_flag(v)) return false; prm_.use_tma = (int)v; }
        else if (k == "lanes") { if (!whole_in(v, 0, kFusedMaxLanes)) return false; prm_.lanes = (int)v; }
        else if (k == "median_filtering") { if (!(v == 0 || v == 1 || v == 3 || v == 5)) return false; prm_.median_filtering = (int)v; }
        else if (k == "median_interval") { if (!whole_in(v, 1, INT_MAX)) return false; prm_.median_interval = (int)v; }
        else if (k == "use_initial_flow") { if (!is_flag(v)) return false; prm_.use_initial_flow = (int)v; }
        else if (k == "gamma") { if (!(std::isfinite(v) && v >= 0)) return false; prm_.gamma = v; }
        else return false;
        return true;
    }
    bool get_param(const std::string &k, double *v) const override {
        if (k == "tau") *v = prm_.tau;
        else if (k == "lambda") *v = prm_.lambda;
        else if (k == "theta") *v = prm_.theta;
        else if (k == "nscales") *v = prm_.nscales;
        else if (k == "warps") *v = prm_.warps;
        else if (k == "epsilon") *v = prm_.epsilon;
        else if (k == "iterations") *v = prm_.iterations;
        else if (k == "scale_step") *v = prm_.scale_step;
        else if (k == "fused") *v = prm_.fused;
        else if (k == "fused_k") *v = prm_.fused_k;
        else if (k == "time_kernels") *v = prm_.time_kernels;
        else if (k == "use_tma") *v = prm_.use_tma;
        else if (k == "lanes") *v = prm_.lanes;
        else if (k == "median_filtering") *v = prm_.median_filtering;
        else if (k == "median_interval") *v = prm_.median_interval;
        else if (k == "use_initial_flow") *v = prm_.use_initial_flow;
        else if (k == "gamma") *v = prm_.gamma;
        else return false;
        return true;
    }

    // A.1: level sizes = round-half-even(dim * scaleStep); a level with cols<16 || rows<16 is dropped.
    int level_geometry(int w, int h, LevelGeom *lv) const {
        int n = 1;
        lv[0] = {w, h, round_up(w, 32)};
        for (int s = 1; s < prm_.nscales; ++s) {
            const int nw = (int)std::nearbyint((double)lv[s - 1].w * prm_.scale_step);
            const int nh = (int)std::nearbyint((double)lv[s - 1].h * prm_.scale_step);
            if (nw < 16 || nh < 16) break;
            lv[s] = {nw, nh, round_up(nw, 32)};
            n = s + 1;
        }
        return n;
    }

    void prepare_frames(int n, const uint8_t *const *srcs, size_t pitch_bytes, int w, int h, const int *slots, cudaStream_t s) override {
        LevelGeom lv[kMaxScales];
        const int nl = level_geometry(w, h, lv);
        const float finv = (float)(1.0 / prm_.scale_step);  // dsize empty => fx = float(1/scaleStep)
        for (int f0 = 0; f0 < n; f0 += kMaxFrameBatch) {
            const int nf = std::min(kMaxFrameBatch, n - f0);
            FramePtrs fp{};
            for (int i = 0; i < nf; ++i) {
                fp.src[i] = srcs[f0 + i];
                fp.base[i] = slots_.at(slots[f0 + i]);
            }
            launch_u8_to_f32_batch(fp, nf, pitch_bytes, w, h, lv[0].pitch, s);
            ++launches;
            size_t off = 0;
            for (int l = 1; l < nl; ++l) {
                const size_t next = off + level_stride(l - 1);
                launch_resize_linear_batch(fp, nf, off, lv[l - 1].w, lv[l - 1].h, lv[l - 1].pitch, next, lv[l].w, lv[l].h, lv[l].pitch, finv, finv, s);
                ++launches;
                off = next;
            }
        }
    }

    // pairs per fused launch.  Utilisation model: a lane of G = SMs / B CTAs visits tiles(level) tiles
    // in ceil(tiles / G) rounds; weight the levels by where the iterations are (the coarsest scale runs
    // most of them), pick the B with the fewest idle CTA-rounds.
    static constexpr double kResidentChunkCost = 0.85;  // time of a resident chunk relative to a streamed one (DESIGN §4.4)
    int max_concurrent_pairs(int w, int h) override {
        if (!prm_.fused) return 1;
        if (prm_.lanes > 0) return prm_.lanes;
        LevelGeom lv[kMaxScales];
        const int n = level_geometry(w, h, lv);
        const int sms = fused_cta_slots(device_);
        const int hy = prm_.fused_k, hx = (hy + 3) & ~3;
        // lanes are sized for the handle's MAXIMUM frame: keep their total workspace under 8 GB
        const size_t lane_bytes = 4 * Slab::padded(pyr_elems_, 4) + 14 * Slab::padded(plane_elems_, 4) + (prm_.gamma > 0 ? gamma_lane_bytes() : 0);
        const int mem_cap = (int)std::max<size_t>(1, (size_t(8) << 30) / std::max<size_t>(lane_bytes, 1));
        const int maxB = std::min(kFusedMaxLanes, mem_cap);
        double util[kFusedMaxLanes + 1] = {};
        double best_u = 0;
        for (int B = 1; B <= maxB; ++B) {
            const int G = sms / B;
            if (G < 1) break;
            double num = 0, den = 0;
            for (int l = 0; l < n; ++l) {
                const double wgt = l == n - 1 ? 7.0 : (l == n - 2 ? 1.5 : 1.0);
                const int tiles = fused_tiles_along(lv[l].w, kFusedTileW, hx) * fused_tiles_along(lv[l].h, kFusedTileH, hy);
                const int rounds = (tiles + G - 1) / G;
                num += wgt * tiles;
                // a level with a CTA per tile keeps its tiles on chip across chunks (tvl1_fused.cu, level_resident): its chunks
                // skip most of the tile load and store
                den += wgt * (double)rounds * G * (tiles <= G ? kResidentChunkCost : 1.0);
            }
            util[B] = num / den * (double)(G * B) / sms;
            best_u = std::max(best_u, util[B]);
        }
        // the smallest lane count within 5 % of the best modelled utilisation: more lanes than needed cost workspace, L2 hits
        // (7.9 -> 10.8 GB of DRAM traffic per 1080p pair from 7 to 16 lanes) and a longer un-overlapped download of the last group
        int best = 1;
        for (int B = 1; B <= maxB; ++B)
            if (util[B] >= 0.95 * best_u) {
                best = B;
                break;
            }
        return best;
    }

    void solve_batch(const PairJob *jobs, int count, int w, int h, cudaStream_t s) override {
        LevelGeom lv[kMaxScales];
        const int n = level_geometry(w, h, lv);
        last_nscales_ = n;
        last_warps_ = prm_.warps;
        std::memcpy(last_lv_, lv, sizeof(lv));
        if (!prm_.fused) {
            for (int i = 0; i < count; ++i) {
                float *flow = jobs[i].flow_xy;
                size_t pitch = jobs[i].flow_pitch_bytes;
                const bool init = jobs[i].init_x != nullptr;
                if (init) load_initial_flow(jobs + i, 1, lv, n, s);
                if (jobs[i].fx) {  // the merge writes the planes straight from u1 / u2
                    solve_unfused(jobs[i].slot_a, jobs[i].slot_b, lv, n, nullptr, 0, s, jobs[i].fx, jobs[i].fy, jobs[i].f_pitch, init);
                    continue;
                }
                if (!flow) {  // quantised output only: the float2 field lives in an engine-owned scratch plane
                    if (!unfused_scratch_) DFB_CUDA(cudaMalloc(&unfused_scratch_, (size_t)max_w_ * max_h_ * 2 * sizeof(float)));
                    flow = unfused_scratch_;
                    pitch = (size_t)w * 2 * sizeof(float);
                }
                solve_unfused(jobs[i].slot_a, jobs[i].slot_b, lv, n, flow, pitch, s, nullptr, nullptr, 0, init);
                if (jobs[i].bound > 0) {  // the reference's structure: a separate pass over the finished field
                    launch_quantise(flow, pitch, lv[0].w, lv[0].h, jobs[i].bound, jobs[i].qx, jobs[i].qy, jobs[i].q_pitch, s);
                    ++launches;
                }
            }
            return;
        }
        const int B = std::min(max_concurrent_pairs(w, h), kFusedMaxLanes);
        for (int i = 0; i < count; i += B) solve_fused(jobs + i, std::min(B, count - i), lv, n, s);
    }

    void phase_ns(uint64_t *out) override {
        if (stats_pending_) DFB_CUDA(cudaEventSynchronize(stats_event_));
        for (int i = 0; i < 32; ++i) out[i] = prm_.fused ? lanes_[last_lane_].host_ctl->prof[i] : 0;
    }
    void tvl1_stats(dfb_tvl1_stats *out) override {
        *out = dfb_tvl1_stats{};
        if (stats_pending_) {  // fused engine: the log was written by the kernel into mapped host memory
            DFB_CUDA(cudaEventSynchronize(stats_event_));
            std::memcpy(last_iters_, pair_log_ + (size_t)last_log_slot_ * kLogInts, sizeof(last_iters_));
            stats_pending_ = false;
        }
        pixel_iters = unfused_px_iters_;
        pixel_chunks = 0;
        for (auto &l : lanes_) {
            pixel_iters += l.host_ctl->px_iters_total;
            pixel_chunks += l.host_ctl->px_chunks_total;
        }
        out->nscales = last_nscales_;
        out->warps = last_warps_;
        for (int s = 0; s < last_nscales_; ++s) {
            out->level_w[s] = last_lv_[s].w;
            out->level_h[s] = last_lv_[s].h;
        }
        std::memcpy(out->iters, last_iters_, sizeof(last_iters_));
    }

    void begin_batch() override { pair_log_count_ = 0; }
    std::string fault_info() override {
        for (size_t i = 0; i < lanes_.size(); ++i) {
            const volatile unsigned *st = lanes_[i].host_ctl->stall;
            if (st[0])
                return "k_tvl1_pair grid-barrier watchdog: CTA " + std::to_string(st[1]) + " (lane " + std::to_string(st[5]) + ", " +
                       std::to_string(st[4]) + " CTAs per lane) waited for arrival count " + std::to_string(st[2]) + ", saw " + std::to_string(st[3]);
        }
        return {};
    }
    bool pair_stats(int idx, dfb_tvl1_stats *out) override {
        *out = dfb_tvl1_stats{};
        if (idx < 0 || idx >= pair_log_count_ || idx < pair_log_count_ - kPairLog) return false;
        if (stats_pending_) DFB_CUDA(cudaEventSynchronize(stats_event_));
        out->nscales = last_nscales_;
        out->warps = last_warps_;
        for (int s = 0; s < last_nscales_; ++s) {
            out->level_w[s] = last_lv_[s].w;
            out->level_h[s] = last_lv_[s].h;
        }
        std::memcpy(out->iters, pair_log_ + (size_t)(idx % kPairLog) * kLogInts, sizeof(out->iters));
        return true;
    }

    // Test hook (dfb_debug_run_kernel "tvl1_*"): one phase of the fused pair kernel on host planes, run by k_tvl1_stage on the
    // engine's own lanes (lane i: frame slots 2i / 2i + 1), tensor maps and level geometry.  Every plane stacks one plane per
    // lane along its rows.  Workspace planes are filled with a finite poison value (0x41414141 = 12.08f) before the inputs are
    // uploaded, so a stage that reads padding, halo or another lane's rows shows up in the image pixels.
    bool debug_run(const std::string &k, const float *const *in, int n_in, float *const *out, int n_out, int w, int h, const double *scalars,
                   int n_scalars, double *scalar_out) override {
        if (k == "tvl1_initial_flow") return debug_initial_flow(k, in, n_in, out, n_out, w, h, scalars, n_scalars);
        static const struct {
            const char *name;
            int stage, n_in, n_out, n_sc;
        } kStages[] = {{"tvl1_level_start", kFusedStageLevelStart, 3, 8, 2}, {"tvl1_warp", kFusedStageWarp, 6, 4, 1},
                       {"tvl1_gq", kFusedStageGq, 1, 1, 1},        {"tvl1_chunks", kFusedStageChunks, 10, 6, 6},
                       {"tvl1_upsample", kFusedStageUpsample, 2, 2, 3}, {"tvl1_merge", kFusedStageMerge, 2, 2, 2},
                       {"tvl1_median", kFusedStageMedian, 2, 2, 2}};
        int si = -1;
        for (int i = 0; i < (int)(sizeof(kStages) / sizeof(kStages[0])); ++i)
            if (k == kStages[i].name) si = i;
        if (si < 0) return false;
        const auto &st = kStages[si];
        if (n_in != st.n_in || n_out != st.n_out)
            throw std::runtime_error(k + ": expects " + std::to_string(st.n_in) + " inputs and " + std::to_string(st.n_out) + " outputs");
        auto sc = [&](int i, double dflt) { return i < n_scalars ? scalars[i] : dflt; };
        // lanes is the last scalar, also when a call passes more scalars than the stage reads
        const int nb = n_scalars >= st.n_sc ? (int)scalars[n_scalars - 1] : 1;
        if (nb < 1 || nb > kFusedParamLanes || h % nb) throw std::runtime_error(k + ": lanes must be in [1, 16] and divide the height");
        const int ph = h / nb;
        // level 0 = the planes' size; the upsample runs from level 1 (its inputs) to level 0 (its destination)
        LevelGeom lv[2];
        int nl = 1;
        if (st.stage == kFusedStageUpsample) {
            const int dw = (int)sc(0, 0), dh = (int)sc(1, 0);
            lv[0] = {dw, dh, round_up(std::max(dw, 1), 32)};
            lv[1] = {w, ph, round_up(w, 32)};
            nl = 2;
        } else {
            lv[0] = {w, ph, round_up(w, 32)};
        }
        for (int l = 0; l < nl; ++l)
            if (lv[l].w < 1 || lv[l].h < 1 || (size_t)lv[l].pitch * (lv[l].h + 1) > max_lv_elems_[l])
                throw std::runtime_error(k + ": plane size outside the handle's level " + std::to_string(l));
        const int level = nl - 1;
        const int slots = fused_cta_slots(device_);
        int G = st.stage == kFusedStageChunks ? (int)sc(3, 0) : 0;
        if (G == 0) G = std::max(1, slots / nb);
        if (G < 1 || G * nb > slots) throw std::runtime_error(k + ": G x lanes must be in [1, " + std::to_string(slots) + "]");
        const int kk = (int)sc(0, 1), nch = (int)sc(1, 1);
        if (st.stage == kFusedStageChunks && (kk < 1 || kk > kFusedMaxK || 2 * kk >= kFusedTileH || nch < 1))
            throw std::runtime_error(k + ": kk must be in [1, " + std::to_string(kFusedMaxK) + "] and n >= 1");
        const int bound = st.stage == kFusedStageMerge ? (int)sc(0, 0) : 0;
        const int median_k = st.stage == kFusedStageMedian ? (int)sc(0, 0) : 0;
        if (st.stage == kFusedStageMedian && median_k != 3 && median_k != 5) throw std::runtime_error(k + ": the window must be 3 or 5");

        DFB_CUDA(cudaDeviceSynchronize());  // nothing of an earlier asynchronous call may still use the slots or lanes
        const cudaStream_t s = nullptr;
        ensure_slots(2 * nb);
        ensure_lanes(nb);
        const Tvl1Params keep = prm_;
        if (st.stage == kFusedStageChunks) prm_.use_tma = sc(4, 1) != 0;
        std::vector<void *> scratch;
        FusedJob jobs[kFusedParamLanes];
        for (int i = 0; i < nb; ++i) {
            PairJob pj{2 * i, 2 * i + 1, nullptr, 0};
            if (st.stage == kFusedStageMerge) {  // the epilogue's destination: float2 rows, or two uint8 planes
                void *p = nullptr;
                DFB_CUDA(cudaMalloc(&p, (size_t)w * ph * 8));
                scratch.push_back(p);
                pj.flow_xy = static_cast<float *>(p);
                pj.flow_pitch_bytes = (size_t)w * 8;
                pj.bound = bound;
                pj.qx = static_cast<uint8_t *>(p);
                pj.qy = pj.qx + (size_t)w * ph;
                pj.q_pitch = (size_t)w;
            }
            fill_job(jobs[i], lanes_[i], pj, lv, nl);
            jobs[i].median_k = median_k;
        }
        prm_ = keep;

        auto plane = [&](const float *p, int l) { return Plane{const_cast<float *>(p), lv[l].w, lv[l].h, lv[l].pitch}; };
        constexpr int kPoison = 0x41;
        const int cur_out = st.stage == kFusedStageChunks ? nch & 1 : 0;
        std::vector<std::vector<Plane>> outs(nb);
        for (int i = 0; i < nb; ++i) {
            const FusedJob &J = jobs[i];
            const FusedLevel &L = J.lv[level];
            for (int b = 0; b < 2; ++b) {  // every workspace plane the phase may touch starts poisoned
                fill_plane(plane(J.lv[0].u1[b], 0), kPoison);
                fill_plane(plane(J.lv[0].u2[b], 0), kPoison);
                for (int q = 0; q < 4; ++q) fill_plane(plane(J.p[b][q], 0), kPoison);
            }
            for (const float *p : {J.I1x, J.I1y, J.I1wx, J.I1wy, J.grad, J.rho_c}) fill_plane(plane(p, 0), kPoison);
            std::vector<Plane> ins;
            switch (st.stage) {
            case kFusedStageLevelStart:
                ins = {plane(L.I1, 0), plane(L.u1[0], 0), plane(L.u2[0], 0)};
                outs[i] = {plane(J.I1x, 0), plane(J.I1y, 0), plane(J.p[0][0], 0), plane(J.p[0][1], 0), plane(J.p[0][2], 0), plane(J.p[0][3], 0),
                           plane(L.u1[0], 0), plane(L.u2[0], 0)};
                break;
            case kFusedStageWarp:
                ins = {plane(L.I0, 0), plane(L.I1, 0), plane(J.I1x, 0), plane(J.I1y, 0), plane(L.u1[0], 0), plane(L.u2[0], 0)};
                outs[i] = {plane(J.I1wx, 0), plane(J.I1wy, 0), plane(J.grad, 0), plane(J.rho_c, 0)};
                break;
            case kFusedStageGq:
                ins = {plane(J.grad, 0)};
                outs[i] = ins;
                break;
            case kFusedStageChunks:
                ins = {plane(J.I1wx, 0), plane(J.I1wy, 0), plane(J.grad, 0), plane(J.rho_c, 0), plane(L.u1[0], 0), plane(L.u2[0], 0),
                       plane(J.p[0][0], 0), plane(J.p[0][1], 0), plane(J.p[0][2], 0), plane(J.p[0][3], 0)};
                outs[i] = {plane(L.u1[cur_out], 0), plane(L.u2[cur_out], 0)};
                for (int q = 0; q < 4; ++q) outs[i].push_back(plane(J.p[cur_out][q], 0));
                break;
            case kFusedStageUpsample:
                ins = {plane(L.u1[0], 1), plane(L.u2[0], 1)};
                outs[i] = {plane(J.lv[0].u1[0], 0), plane(J.lv[0].u2[0], 0)};
                break;
            case kFusedStageMedian:
                ins = {plane(L.u1[0], 0), plane(L.u2[0], 0)};
                outs[i] = {plane(L.u1[1], 0), plane(L.u2[1], 0)};
                break;
            default:  // merge
                ins = {plane(L.u1[0], 0), plane(L.u2[0], 0)};
                break;
            }
            for (int q = 0; q < n_in; ++q) upload_rows(ins[q], in[q], i * ins[q].h, kPoison);
        }
        FusedBatch batch{};
        batch.njobs = nb;
        batch.group = G;
        batch.host_jobs = jobs;
        FusedStageArgs a{st.stage, level, (int)sc(0, 0) != 0, kk, nch, sc(2, 0) != 0};
        if (st.stage == kFusedStageChunks) {  // the gradient plane as the inner loop reads it
            FusedStageArgs g = a;
            g.stage = kFusedStageGq;
            launch_tvl1_stage(batch, g, s);
        }
        launch_tvl1_stage(batch, a, s);
        DFB_CUDA(cudaDeviceSynchronize());
        for (int i = 0; i < nb; ++i) {
            if (st.stage != kFusedStageMerge) {
                for (int q = 0; q < n_out; ++q) download_rows(out[q], outs[i][q], i * outs[i][q].h);
                continue;
            }
            const size_t npx = (size_t)w * ph;
            if (bound > 0) {
                std::vector<uint8_t> q(2 * npx);
                DFB_CUDA(cudaMemcpy(q.data(), scratch[i], 2 * npx, cudaMemcpyDeviceToHost));
                for (size_t j = 0; j < npx; ++j) {
                    out[0][i * npx + j] = q[j];
                    out[1][i * npx + j] = q[npx + j];
                }
            } else {
                std::vector<float> f(2 * npx);
                DFB_CUDA(cudaMemcpy(f.data(), scratch[i], 2 * npx * sizeof(float), cudaMemcpyDeviceToHost));
                for (size_t j = 0; j < npx; ++j) {
                    out[0][i * npx + j] = f[2 * j];
                    out[1][i * npx + j] = f[2 * j + 1];
                }
            }
        }
        for (void *p : scratch) DFB_CUDA(cudaFree(p));
        if (st.stage == kFusedStageChunks && a.check && scalar_out)
            for (int i = 0; i < nb; ++i) scalar_out[i] = lanes_[i].host_ctl->error;
        // the hook's level geometry (an upsample's source level comes from the caller) is not the handle's pyramid: the next
        // pair re-encodes its tensor maps
        for (int i = 0; i < nb; ++i) lanes_[i].tmap_w = 0;
        return true;
    }

  private:
    // Test hook "tvl1_initial_flow": load_initial_flow on `lanes` lanes (scalars {step, pitch, lanes}), lane i starting from
    // rows [i * h / lanes, (i + 1) * h / lanes) of the two input planes, laid out on the device as the calls pass it: step 2 a
    // float2 field, step 1 two planes, rows `pitch` floats apart (0: dense).  out[0] / out[1]: every lane's u1pyr[0] / u2pyr[0]
    // at the handle's nscales / scale_step, level after level, each level the lanes' dense planes stacked along the rows.  The lane pyramids and the start
    // buffers' padding hold NaN first, so a read of padding or a pyramid left unwritten shows; the pyramids are zero after.
    bool debug_initial_flow(const std::string &k, const float *const *in, int n_in, float *const *out, int n_out, int w, int h,
                            const double *scalars, int n_scalars) {
        auto sc = [&](int i, double dflt) { return i < n_scalars ? scalars[i] : dflt; };
        const int step = (int)sc(0, 2), nb = (int)sc(2, 1);
        if (n_in != 2) throw std::runtime_error(k + ": expects 2 inputs");
        if (step != 1 && step != 2) throw std::runtime_error(k + ": step must be 1 or 2");
        if (nb < 1 || nb > kFusedMaxLanes || h % nb) throw std::runtime_error(k + ": lanes must be in [1, 64] and divide the height");
        const int ph = h / nb;
        const size_t row = (size_t)w * step, pitch = sc(1, 0) > 0 ? (size_t)sc(1, 0) : row;
        if (pitch < row) throw std::runtime_error(k + ": pitch smaller than a row");
        LevelGeom lv[kMaxScales];
        const int n = level_geometry(w, ph, lv);
        if (n_out != 2) throw std::runtime_error(k + ": expects 2 outputs");
        for (int l = 0; l < n; ++l)
            if (w < 1 || (size_t)lv[l].pitch * (lv[l].h + 1) > max_lv_elems_[l])
                throw std::runtime_error(k + ": plane size outside the handle's level " + std::to_string(l));

        DFB_CUDA(cudaDeviceSynchronize());  // nothing of an earlier asynchronous call may still use the lanes
        const cudaStream_t s = nullptr;
        ensure_lanes(nb);
        const size_t pyr_bytes = Slab::padded(pyr_elems_, 4);
        std::vector<DeviceBuffer<float>> bufs(nb);
        std::vector<PairJob> jobs(nb);
        for (int i = 0; i < nb; ++i) {
            DFB_CUDA(cudaMemset(lanes_[i].u1pyr[0], 0xff, pyr_bytes));
            DFB_CUDA(cudaMemset(lanes_[i].u2pyr[0], 0xff, pyr_bytes));
            jobs[i] = PairJob{2 * i, 2 * i + 1, nullptr, 0};
            stage_initial_flow(bufs[i], jobs[i], in[0], in[1], i * ph, w, ph, step, pitch);
        }
        load_initial_flow(jobs.data(), nb, lv, n, s);
        DFB_CUDA(cudaDeviceSynchronize());
        for (int i = 0; i < nb; ++i) {
            size_t off = 0;  // level l's first element in the outputs
            for (int l = 0; l < n; off += (size_t)nb * lv[l].w * lv[l].h, ++l)
                for (int c = 0; c < 2; ++c) {
                    const Plane p = level_plane(c ? lanes_[i].u2pyr[0] : lanes_[i].u1pyr[0], lv, l);
                    download_rows(out[c] + off, p, i * p.h);
                }
            DFB_CUDA(cudaMemset(lanes_[i].u1pyr[0], 0, pyr_bytes));  // as ensure_lanes leaves them
            DFB_CUDA(cudaMemset(lanes_[i].u2pyr[0], 0, pyr_bytes));
        }
        DFB_CUDA(cudaDeviceSynchronize());
        return true;
    }

    int next_log_slot() {
        last_log_slot_ = pair_log_count_ % kPairLog;
        ++pair_log_count_;
        return last_log_slot_;
    }
    Plane level_plane(float *base, const LevelGeom *lv, int l) const {
        size_t off = 0;
        for (int i = 0; i < l; ++i) off += level_stride(i);
        return Plane{base + off, lv[l].w, lv[l].h, lv[l].pitch};
    }
    // slot layout is fixed by the MAX geometry so any smaller frame fits
    size_t level_stride(int l) const { return max_lv_elems_[l]; }

    void allocate() {
        // geometry of the largest frame, with the full default pyramid depth available
        Tvl1Params keep = prm_;
        prm_.nscales = kMaxScales;
        prm_.scale_step = kAllocScaleStep;
        LevelGeom lv[kMaxScales];
        const int n = level_geometry(max_w_, max_h_, lv);
        prm_ = keep;
        pyr_elems_ = 0;
        for (int l = 0; l < kMaxScales; ++l) {
            // +pitch: one spare row so float4 tile reads one row past the image stay inside the slab
            max_lv_elems_[l] = l < n ? (size_t)lv[l].pitch * (lv[l].h + 1) : 0;
            max_lv_elems_[l] = (max_lv_elems_[l] + 63) & ~size_t(63);
            pyr_elems_ += max_lv_elems_[l];
        }
        plane_elems_ = (size_t)lv[0].pitch * (lv[0].h + 1);
        slab_.reserve(kInitialSlots * Slab::padded(pyr_elems_, 4) + (1 << 12));
        carve_slots(slab_, pyr_elems_);
        ensure_lanes(1);
        DFB_CUDA(cudaEventCreateWithFlags(&stats_event_, cudaEventDisableTiming));
        DFB_CUDA(cudaHostAlloc(&pair_log_, sizeof(int) * kLogInts * kPairLog, cudaHostAllocMapped));
        std::memset(pair_log_, 0, sizeof(int) * kLogInts * kPairLog);
        DFB_CUDA(cudaHostGetDevicePointer(&pair_log_dev_, pair_log_, 0));
        // every plane starts finite: padding columns are read (never used) by vectorised kernels
        slab_.zero();
    }

    // per-pair workspace: flow pyramids (ping-pong), gradient / warp planes, dual variables (ping-pong),
    // convergence partials, barrier words and the mapped control block
    struct Lane {
        void *own = nullptr;
        float *u1pyr[2] = {}, *u2pyr[2] = {};
        float *I1x = nullptr, *I1y = nullptr, *I1wx = nullptr, *I1wy = nullptr, *grad = nullptr, *rho_c = nullptr;
        float *p[2][4] = {};
        double *partials = nullptr;
        unsigned *sync = nullptr;
        FusedHostCtl *host_ctl = nullptr, *dev_ctl = nullptr;
        void *tmaps = nullptr;  // device array CUtensorMap[kMaxScales][kFusedMapsPerLevel]
        void *gamma_own = nullptr;  // gamma > 0 (ensure_gamma_lanes): the u3 pyramid and p31 / p32
        float *u3pyr = nullptr, *p3[2] = {};
        int tmap_w = 0, tmap_h = 0, tmap_n = 0;
        double tmap_ss = 0;
    };

    void ensure_lanes(int n) {
        while ((int)lanes_.size() < n) {
            Lane l;
            const size_t pyr = Slab::padded(pyr_elems_, 4), pl = Slab::padded(plane_elems_, 4);
            const size_t bytes = 4 * pyr + 14 * pl + Slab::padded(kMaxPartials, 8) + 256;
            DFB_CUDA(cudaMalloc(&l.own, bytes));
            DFB_CUDA(cudaMemset(l.own, 0, bytes));  // planes start finite: padding is read (never used) by vector loads
            DFB_CUDA(cudaDeviceSynchronize());      // null-stream memset vs the caller's (possibly non-blocking) stream
            char *c = static_cast<char *>(l.own);
            auto take = [&](size_t b) { char *r = c; c += b; return r; };
            for (int b = 0; b < 2; ++b) {
                l.u1pyr[b] = reinterpret_cast<float *>(take(pyr));
                l.u2pyr[b] = reinterpret_cast<float *>(take(pyr));
            }
            l.I1x = reinterpret_cast<float *>(take(pl));
            l.I1y = reinterpret_cast<float *>(take(pl));
            l.I1wx = reinterpret_cast<float *>(take(pl));
            l.I1wy = reinterpret_cast<float *>(take(pl));
            l.grad = reinterpret_cast<float *>(take(pl));
            l.rho_c = reinterpret_cast<float *>(take(pl));
            for (int b = 0; b < 2; ++b)
                for (int k = 0; k < 4; ++k) l.p[b][k] = reinterpret_cast<float *>(take(pl));
            l.partials = reinterpret_cast<double *>(take(Slab::padded(kMaxPartials, 8)));
            l.sync = reinterpret_cast<unsigned *>(take(256));
            DFB_CUDA(cudaHostAlloc(&l.host_ctl, sizeof(FusedHostCtl), cudaHostAllocMapped));
            std::memset(l.host_ctl, 0, sizeof(FusedHostCtl));
            DFB_CUDA(cudaHostGetDevicePointer(&l.dev_ctl, l.host_ctl, 0));
            DFB_CUDA(cudaMalloc(&l.tmaps, (size_t)kMaxScales * kFusedMapsPerLevel * kTensorMapBytes));
            lanes_.push_back(l);
        }
    }

    Plane work(float *p, const LevelGeom &g) const { return Plane{p, g.w, g.h, g.pitch}; }

    // gamma > 0: each lane's u3 pyramid and p31 / p32 planes, allocated when a gamma solve first needs the lane
    size_t gamma_lane_bytes() const { return Slab::padded(pyr_elems_, 4) + 2 * Slab::padded(plane_elems_, 4); }
    void ensure_gamma_lanes(int n) {
        ensure_lanes(n);
        for (int i = 0; i < n; ++i) {
            Lane &l = lanes_[i];
            if (l.gamma_own) continue;
            const size_t pyr = Slab::padded(pyr_elems_, 4), pl = Slab::padded(plane_elems_, 4);
            DFB_CUDA(cudaMalloc(&l.gamma_own, gamma_lane_bytes()));
            DFB_CUDA(cudaMemset(l.gamma_own, 0, gamma_lane_bytes()));  // padding columns are read (never used) by the vector loads
            DFB_CUDA(cudaDeviceSynchronize());  // null-stream memset vs the caller's (possibly non-blocking) stream
            char *c = static_cast<char *>(l.gamma_own);
            l.u3pyr = reinterpret_cast<float *>(c);
            l.p3[0] = reinterpret_cast<float *>(c + pyr);
            l.p3[1] = reinterpret_cast<float *>(c + pyr + pl);
        }
    }

    // use_initial_flow: the initial fields of the pairs jobs[i] that carry one (PairJob::init_x) into lane i's flow pyramid
    // u1pyr[0] / u2pyr[0], enqueued before the solve.  Level 0 is the field as given; level s is resize_linear of level s - 1
    // with the frame pyramid's taps (prepare_frames), times float(scale_step) (DESIGN §1).
    void load_initial_flow(const PairJob *jobs, int count, const LevelGeom *lv, int n, cudaStream_t s) {
        InitFlows f{};
        int m = 0;
        auto flush = [&]() {
            if (m) launch_split_initial_flow(f, m, lv[0].w, lv[0].h, lv[0].pitch, s);
            launches += m ? 1 : 0;
            m = 0;
        };
        for (int i = 0; i < count; ++i) {
            if (!jobs[i].init_x) continue;
            f.x[m] = jobs[i].init_x;
            f.y[m] = jobs[i].init_y;
            f.pitch[m] = jobs[i].init_pitch;
            f.step[m] = jobs[i].init_step;
            f.u1[m] = lanes_[i].u1pyr[0];  // level 0 starts the pyramid
            f.u2[m] = lanes_[i].u2pyr[0];
            if (++m == kMaxInitFlows) flush();
        }
        flush();
        const float finv = (float)(1.0 / prm_.scale_step), mul = (float)prm_.scale_step;
        for (int i = 0; i < count; ++i) {
            if (!jobs[i].init_x) continue;
            for (int l = 1; l < n; ++l) {
                launch_resize_linear(level_plane(lanes_[i].u1pyr[0], lv, l - 1), level_plane(lanes_[i].u1pyr[0], lv, l), finv, finv, mul, s);
                launch_resize_linear(level_plane(lanes_[i].u2pyr[0], lv, l - 1), level_plane(lanes_[i].u2pyr[0], lv, l), finv, finv, mul, s);
                launches += 2;
            }
        }
    }

    // ---- fused = 0: reference launch structure, A.4 state machine on the host ------------------
    // fx set: the merge writes the two float planes fx / fy (PairJob) instead of the float2 field, and flow_xy may be null.
    // init: lane 0's flow pyramid holds the initial flow (load_initial_flow), the coarsest level starts from it.
    void solve_unfused(int slot_a, int slot_b, const LevelGeom *lv, int n, float *flow_xy, size_t flow_pitch_bytes,
                       cudaStream_t s, float *fx = nullptr, float *fy = nullptr, size_t f_pitch = 0, bool init = false) {
        const Tvl1Consts c{(float)(prm_.lambda * prm_.theta), (float)(prm_.tau / prm_.theta), (float)prm_.theta};
        const bool gam = prm_.gamma > 0;
        const float gamma = (float)prm_.gamma;
        if (gam) ensure_gamma_lanes(1);
        std::memset(last_iters_, 0, sizeof(last_iters_));
        Lane &wk = lanes_[0];
        float *I0b = slots_.at(slot_a), *I1b = slots_.at(slot_b);
        for (int l = n - 1; l >= 0; --l) {
            const LevelGeom &g = lv[l];
            const Plane I0 = level_plane(I0b, lv, l), I1 = level_plane(I1b, lv, l);
            const Plane u1 = level_plane(wk.u1pyr[0], lv, l), u2 = level_plane(wk.u2pyr[0], lv, l);
            const Plane I1x = work(wk.I1x, g), I1y = work(wk.I1y, g), I1wx = work(wk.I1wx, g), I1wy = work(wk.I1wy, g);
            const Plane grad = work(wk.grad, g), rho_c = work(wk.rho_c, g);
            const Plane p11 = work(wk.p[0][0], g), p12 = work(wk.p[0][1], g), p21 = work(wk.p[0][2], g), p22 = work(wk.p[0][3], g);
            if (l == n - 1 && !init) {  // useInitialFlow = false
                launch_fill(u1, 0.f, s);
                launch_fill(u2, 0.f, s);
                launches += 2;
            }
            // gamma: u3 starts at 0 on the coarsest level (initial flow or not), p31 / p32 at every scale like p11 .. p22
            Plane u3{}, pg[6] = {p11, p12, p21, p22, {}, {}};
            if (gam) {
                u3 = level_plane(wk.u3pyr, lv, l);
                pg[4] = work(wk.p3[0], g);
                pg[5] = work(wk.p3[1], g);
                if (l == n - 1) {
                    launch_fill(u3, 0.f, s);
                    ++launches;
                }
                launch_fill(pg[4], 0.f, s);
                launch_fill(pg[5], 0.f, s);
                launches += 2;
            }
            launch_centered_gradient(I1, I1x, I1y, s);
            launch_fill(p11, 0.f, s);  // once per scale, not per warp (A.2 step 2)
            launch_fill(p12, 0.f, s);
            launch_fill(p21, 0.f, s);
            launch_fill(p22, 0.f, s);
            launches += 5;
            const double scaled_eps = prm_.epsilon * prm_.epsilon * (double)((long)g.w * g.h);
            const int nblk = estimate_u_blocks(g.w, g.h);
            // the median's destination: this level's plane of the second flow pyramid, which only the fused schedule uses
            const Plane m1 = level_plane(wk.u1pyr[1], lv, l), m2 = level_plane(wk.u2pyr[1], lv, l);
            for (int wi = 0; wi < prm_.warps; ++wi) {
                launch_warp_backward(I0, I1, I1x, I1y, u1, u2, I1wx, I1wy, grad, rho_c, s);
                ++launches;
                double error = DBL_MAX, prev_error = 0.0;
                int it = 0;
                for (; error > scaled_eps && it < prm_.iterations; ++it) {
                    if (prm_.median_k() && it % prm_.median_interval == 0) {  // the A.4 state does not change
                        launch_median(u1, u2, m1, m2, prm_.median_k(), s);
                        ++launches;
                        DFB_CUDA(cudaMemcpy2DAsync(u1.p, (size_t)u1.pitch * 4, m1.p, (size_t)m1.pitch * 4, (size_t)g.w * 4, g.h, cudaMemcpyDeviceToDevice, s));
                        DFB_CUDA(cudaMemcpy2DAsync(u2.p, (size_t)u2.pitch * 4, m2.p, (size_t)m2.pitch * 4, (size_t)g.w * 4, g.h, cudaMemcpyDeviceToDevice, s));
                    }
                    const bool calc_error = prm_.epsilon > 0 && (it & 1) && prev_error < scaled_eps;
                    if (gam)
                        launch_estimate_u_gamma(I1wx, I1wy, grad, rho_c, pg, u1, u2, u3, c, gamma, calc_error ? wk.partials : nullptr, s);
                    else
                        launch_estimate_u(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, u1, u2, c,
                                          calc_error ? wk.partials : nullptr, s);
                    ++launches;
                    if (calc_error) {
                        launch_sum_partials(wk.partials, nblk, &wk.dev_ctl->error, s);
                        ++launches;
                        DFB_CUDA(cudaStreamSynchronize(s));  // the reference syncs here too (stream.waitForCompletion)
                        error = wk.host_ctl->error;
                        prev_error = error;
                    } else {
                        error = DBL_MAX;
                        prev_error -= scaled_eps;
                    }
                    if (gam)
                        launch_estimate_dual_gamma(u1, u2, u3, pg, c, s);
                    else
                        launch_estimate_dual(u1, u2, p11, p12, p21, p22, c, s);
                    ++launches;
                }
                last_iters_[l * prm_.warps + wi] = it;
            }
            if (l > 0) {  // A.2 step 4: explicit dsize => f = float(1 / (dst/src)); then * float(1/scaleStep)
                const float ufx = (float)(1.0 / ((double)lv[l - 1].w / (double)g.w));
                const float ufy = (float)(1.0 / ((double)lv[l - 1].h / (double)g.h));
                const float mul = (float)(1.0 / prm_.scale_step);
                launch_resize_linear(u1, level_plane(wk.u1pyr[0], lv, l - 1), ufx, ufy, mul, s);
                launch_resize_linear(u2, level_plane(wk.u2pyr[0], lv, l - 1), ufx, ufy, mul, s);
                launches += 2;
                if (gam) {  // u3 is an intensity, not a displacement: no 1 / scaleStep
                    launch_resize_linear(u3, level_plane(wk.u3pyr, lv, l - 1), ufx, ufy, 1.0f, s);
                    ++launches;
                }
            }
        }
        launch_merge_flow(level_plane(wk.u1pyr[0], lv, 0), level_plane(wk.u2pyr[0], lv, 0), flow_xy, flow_pitch_bytes, s, fx, fy, f_pitch);
        ++launches;
        stats_pending_ = false;
        std::memcpy(pair_log_ + (size_t)next_log_slot() * kLogInts, last_iters_, sizeof(last_iters_));
        accumulate_pixel_iters();
    }

    // TMA descriptors of the lane's shared-memory-resident planes, rebuilt only when the frame geometry changes
    void ensure_tensor_maps(Lane &wk, const LevelGeom *lv, int n) {
        if (wk.tmap_w == lv[0].w && wk.tmap_h == lv[0].h && wk.tmap_n == n && wk.tmap_ss == prm_.scale_step) return;
        std::vector<char> host((size_t)kMaxScales * kFusedMapsPerLevel * kTensorMapBytes, 0);
        for (int l = 0; l < n; ++l) {
            char *m = host.data() + (size_t)l * kFusedMapsPerLevel * kTensorMapBytes;
            float *planes[kFusedMapsPerLevel] = {wk.I1wx, wk.I1wy, wk.grad, wk.rho_c, level_plane(wk.u1pyr[0], lv, l).p,
                                                 level_plane(wk.u2pyr[0], lv, l).p, level_plane(wk.u1pyr[1], lv, l).p,
                                                 level_plane(wk.u2pyr[1], lv, l).p};
            for (int k = 0; k < kFusedMapsPerLevel; ++k)
                fused_encode_tensor_map(m + (size_t)k * kTensorMapBytes, planes[k], lv[l].w, lv[l].h, lv[l].pitch);
        }
        DFB_CUDA(cudaDeviceSynchronize());  // the previous maps may still be in use by a running launch
        DFB_CUDA(cudaMemcpy(wk.tmaps, host.data(), host.size(), cudaMemcpyHostToDevice));
        wk.tmap_w = lv[0].w;
        wk.tmap_h = lv[0].h;
        wk.tmap_n = n;
        wk.tmap_ss = prm_.scale_step;
    }

    // ---- fused = 1 -------------------------------------------------------------------------------
    // the job description of one lane: pair (slot_a -> slot_b) over the n levels lv, with the handle's parameters
    void fill_job(FusedJob &job, Lane &wk, const PairJob &pj, const LevelGeom *lv, int n) {
        job = FusedJob{};
        job.nscales = n;
        job.warps = prm_.warps;
        job.iterations = prm_.iterations;
        job.epsilon = prm_.epsilon;
        job.k = prm_.fused_k;
        job.use_tma = prm_.use_tma;
        job.median_k = prm_.median_k();
        job.median_interval = prm_.median_interval;
        job.init_flow = pj.init_x != nullptr;
        if (prm_.use_tma) ensure_tensor_maps(wk, lv, n);
        job.tmaps = wk.tmaps;
        job.c = Tvl1Consts{(float)(prm_.lambda * prm_.theta), (float)(prm_.tau / prm_.theta), (float)prm_.theta};
        job.up_mul = (float)(1.0 / prm_.scale_step);
        for (int l = 0; l < n; ++l) {
            FusedLevel &L = job.lv[l];
            L.w = lv[l].w;
            L.h = lv[l].h;
            L.pitch = lv[l].pitch;
            L.I0 = level_plane(slots_.at(pj.slot_a), lv, l).p;
            L.I1 = level_plane(slots_.at(pj.slot_b), lv, l).p;
            for (int b = 0; b < 2; ++b) {
                L.u1[b] = level_plane(wk.u1pyr[b], lv, l).p;
                L.u2[b] = level_plane(wk.u2pyr[b], lv, l).p;
            }
            if (l > 0) {
                L.up_fx = (float)(1.0 / ((double)lv[l - 1].w / (double)lv[l].w));
                L.up_fy = (float)(1.0 / ((double)lv[l - 1].h / (double)lv[l].h));
            }
        }
        job.I1x = wk.I1x;
        job.I1y = wk.I1y;
        job.I1wx = wk.I1wx;
        job.I1wy = wk.I1wy;
        job.grad = wk.grad;
        job.rho_c = wk.rho_c;
        for (int b = 0; b < 2; ++b)
            for (int k = 0; k < 4; ++k) job.p[b][k] = wk.p[b][k];
        job.partials = wk.partials;
        job.sync = wk.sync;
        job.ctl = wk.dev_ctl;
        job.flow_xy = pj.flow_xy;
        job.flow_pitch_bytes = pj.flow_pitch_bytes;
        job.bound = pj.bound;
        job.qx = pj.qx;
        job.qy = pj.qy;
        job.q_pitch = pj.q_pitch;
        job.fx = pj.fx;
        job.fy = pj.fy;
        job.f_pitch = pj.f_pitch;
    }

    void solve_fused(const PairJob *jobs, int count, const LevelGeom *lv, int n, cudaStream_t s) {
        ensure_lanes(count);
        FusedBatch batch{};
        batch.njobs = count;
        batch.group = std::max(1, fused_cta_slots(device_) / count);
        // job descriptions: filled in a pinned host slot of a small ring, copied to its device twin on the launch stream
        if (!job_ring_h_[0]) {
            for (int r = 0; r < kJobRing; ++r) {
                DFB_CUDA(cudaHostAlloc(&job_ring_h_[r], sizeof(FusedJob) * kFusedMaxLanes, cudaHostAllocDefault));
                DFB_CUDA(cudaMalloc(&job_ring_d_[r], sizeof(FusedJob) * kFusedMaxLanes));
                DFB_CUDA(cudaEventCreateWithFlags(&job_ring_ev_[r], cudaEventDisableTiming));
            }
        }
        const int jr = job_ring_next_++ % kJobRing;
        if (job_ring_next_ > kJobRing) DFB_CUDA(cudaEventSynchronize(job_ring_ev_[jr]));  // the copy out of this host slot has run (no-op if never recorded)
        FusedJob *host_jobs = job_ring_h_[jr];
        for (int i = 0; i < count; ++i) {
            fill_job(host_jobs[i], lanes_[i], jobs[i], lv, n);
            host_jobs[i].iters_log = pair_log_dev_ + (size_t)next_log_slot() * kLogInts;
        }
        load_initial_flow(jobs, count, lv, n, s);
        // one CTA per SM at most: the tile counts of the largest level bound the useful group size
        const int hx = 4, hy = 1;
        const int max_tiles = fused_tiles_along(lv[0].w, kFusedTileW, hx) * fused_tiles_along(lv[0].h, kFusedTileH, hy);
        batch.group = std::max(1, std::min(batch.group, max_tiles));
        if (prm_.time_kernels) timer_.begin(s);
        if (count > kFusedParamLanes) {  // too many for the parameter bank: through the device-memory ring
            DFB_CUDA(cudaMemcpyAsync(job_ring_d_[jr], host_jobs, sizeof(FusedJob) * count, cudaMemcpyHostToDevice, s));
            DFB_CUDA(cudaEventRecord(job_ring_ev_[jr], s));
        }
        batch.jobs = job_ring_d_[jr];
        batch.host_jobs = host_jobs;
        if (prm_.gamma > 0) {  // the gamma kernel: its planes travel beside the jobs
            ensure_gamma_lanes(count);
            if (!gamma_params_) gamma_params_.reset(new FusedGamma());
            FusedGamma &gm = *gamma_params_;
            gm.gamma = (float)prm_.gamma;
            for (int i = 0; i < count; ++i) {
                for (int l = 0; l < n; ++l) gm.lane[i].u3[l] = level_plane(lanes_[i].u3pyr, lv, l).p;
                gm.lane[i].p31 = lanes_[i].p3[0];
                gm.lane[i].p32 = lanes_[i].p3[1];
            }
            launches += launch_tvl1_fused(batch, device_, s, &gm);
        } else {
            launches += launch_tvl1_fused(batch, device_, s);
        }
        if (prm_.time_kernels) timer_.end(s, 1, count);
        last_lane_ = count - 1;
        DFB_CUDA(cudaEventRecord(stats_event_, s));
        stats_pending_ = true;
    }

    void accumulate_pixel_iters() {
        for (int l = 0; l < last_nscales_; ++l)
            for (int wi = 0; wi < prm_.warps; ++wi)
                unfused_px_iters_ += (uint64_t)last_iters_[l * prm_.warps + wi] * (uint64_t)last_lv_[l].w * last_lv_[l].h;
    }
    void reset_counters() override {
        if (stats_pending_) {
            cudaEventSynchronize(stats_event_);
            stats_pending_ = false;
        }
        FlowAlgorithm::reset_counters();
        unfused_px_iters_ = 0;
        for (auto &l : lanes_) {
            l.host_ctl->px_iters_total = 0;
            l.host_ctl->px_chunks_total = 0;
        }
    }
    std::unique_ptr<FusedGamma> gamma_params_;  // copied into the launch's parameters
    uint64_t unfused_px_iters_ = 0;
    float *unfused_scratch_ = nullptr;
    static constexpr int kJobRing = 8;
    FusedJob *job_ring_h_[kJobRing] = {}, *job_ring_d_[kJobRing] = {};
    cudaEvent_t job_ring_ev_[kJobRing] = {};
    long job_ring_next_ = 0;

    static constexpr size_t kMaxPartials = 1 << 16;

    int device_, max_w_, max_h_;
    Tvl1Params prm_;
    Slab slab_;
    size_t max_lv_elems_[kMaxScales] = {};
    size_t pyr_elems_ = 0, plane_elems_ = 0;
    std::vector<Lane> lanes_;
    int last_lane_ = 0;
    // iteration logs of the last kPairLog pairs, written by the kernel into mapped host memory
    static constexpr int kPairLog = 256, kLogInts = 16 * 16;
    int *pair_log_ = nullptr, *pair_log_dev_ = nullptr;
    int pair_log_count_ = 0, last_log_slot_ = 0;
    cudaEvent_t stats_event_ = nullptr;
    bool stats_pending_ = false;
    int last_nscales_ = 0, last_warps_ = 0;  // the log layout of the most recent call: a later set() does not change it
    LevelGeom last_lv_[kMaxScales] = {};
    int last_iters_[16 * 16] = {};
};

}  // namespace

std::unique_ptr<FlowAlgorithm> make_tvl1(int device, int max_w, int max_h) {
    return std::unique_ptr<FlowAlgorithm>(new Tvl1(device, max_w, max_h));
}

}  // namespace dfb
