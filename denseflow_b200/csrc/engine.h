// engine.h — host-side engine objects behind the C ABI (include/denseflow_b200.h).
// FlowEngine is the replacement for the cv::cuda::DenseOpticalFlow object the reference creates at
// /root/reference/src/denseflow_gpu.cpp:299-301 and calls at :327/:329.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/denseflow_b200.h"
#include "common.cuh"

namespace dfb {

struct LevelGeom {
    int w, h, pitch;
};

// Algorithm back-end working on device buffers. One frame "slot" holds everything that depends on
// a single frame (its fp32 pyramid), so a frame shared by two consecutive pairs is prepared once.
class FlowAlgorithm {
  public:
    virtual ~FlowAlgorithm() = default;
    virtual const char *name() const = 0;
    virtual int num_slots() const = 0;
    virtual void ensure_slots(int n) = 0;
    // per-frame work: u8 -> fp32 (+ pyramid)
    virtual void prepare_frame(const uint8_t *src, size_t pitch_bytes, int w, int h, int slot, cudaStream_t s) = 0;
    // several frames of one size at once (engines whose per-frame stages are launch-latency-bound batch them)
    virtual void prepare_frames(int n, const uint8_t *const *srcs, size_t pitch_bytes, int w, int h, const int *slots, cudaStream_t s) {
        for (int i = 0; i < n; ++i) prepare_frame(srcs[i], pitch_bytes, w, h, slots[i], s);
    }
    // per-pair work: flow(slot_a -> slot_b) into interleaved float2 rows
    virtual void solve(int slot_a, int slot_b, int w, int h, float *flow_xy, size_t flow_pitch_bytes,
                       cudaStream_t s) = 0;
    // several independent pairs at once (the fused tvl1 engine runs them side by side on disjoint SM groups)
    struct PairJob {
        int slot_a, slot_b;
        float *flow_xy;
        size_t flow_pitch_bytes;
        // bound > 0: the merge epilogue writes convertFlowToImage's two uint8 planes (src/common.cpp:4-16, bounds -bound /
        // +bound) to qx / qy (row pitch q_pitch bytes) INSTEAD of the float2 field (SURVEY §8 f1); flow_xy may then be null
        // for the fused tvl1 and Farneback engines (the unfused tvl1 schedule still needs it as scratch)
        int bound = 0;
        uint8_t *qx = nullptr, *qy = nullptr;
        size_t q_pitch = 0;
    };
    virtual int max_concurrent_pairs(int w, int h) { (void)w; (void)h; return 1; }
    // after a CUDA error: what the engine's own watchdogs recorded (empty if nothing)
    virtual std::string fault_info() { return {}; }
    virtual void solve_batch(const PairJob *jobs, int n, int w, int h, cudaStream_t s) {
        for (int i = 0; i < n; ++i) solve(jobs[i].slot_a, jobs[i].slot_b, w, h, jobs[i].flow_xy, jobs[i].flow_pitch_bytes, s);
    }
    virtual bool set_param(const std::string &name, double v) = 0;
    virtual bool get_param(const std::string &name, double *v) const = 0;
    virtual void tvl1_stats(dfb_tvl1_stats *out) { *out = dfb_tvl1_stats{}; }
    // per-pair iteration logs of the most recent batch call: begin_batch() restarts the numbering
    virtual void begin_batch() {}
    virtual bool pair_stats(int pair_index, dfb_tvl1_stats *out) { (void)pair_index; *out = dfb_tvl1_stats{}; return false; }
    virtual void phase_ns(uint64_t *out) { for (int i = 0; i < 32; ++i) out[i] = 0; }
    virtual void reset_counters() { launches = 0; pixel_iters = 0; pixel_chunks = 0; }
    virtual void kernel_timing(uint64_t *launches_, uint64_t *ns, uint64_t *pairs) { *launches_ = *ns = *pairs = 0; }
    // test hook behind dfb_debug_run_kernel: run one stage of this engine, through its own launch code and buffers, on dense
    // host planes (w x h floats each).  Returns false when `kernel` is not one of the engine's stages.
    virtual bool debug_run(const std::string &kernel, const float *const *in, int n_in, float *const *out, int n_out, int w, int h,
                           const double *scalars, int n_scalars) {
        (void)kernel; (void)in; (void)n_in; (void)out; (void)n_out; (void)w; (void)h; (void)scalars; (void)n_scalars;
        return false;
    }
    uint64_t launches = 0;     // kernels launched
    uint64_t pixel_iters = 0;  // tvl1: sum of level pixels over executed inner iterations
    uint64_t pixel_chunks = 0; // fused tvl1: sum of level pixels over tile visits (k iterations each)
};

std::unique_ptr<FlowAlgorithm> make_tvl1(int device, int max_w, int max_h);
std::unique_ptr<FlowAlgorithm> make_farneback(int device, int max_w, int max_h);

}  // namespace dfb
