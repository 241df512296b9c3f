// engine.h — host-side engine objects behind the C ABI (include/denseflow_b200.h).
// FlowEngine is the replacement for the cv::cuda::DenseOpticalFlow object the reference creates at
// /root/reference/src/denseflow_gpu.cpp:299-301 and calls at :327/:329.
#pragma once

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <deque>
#include <memory>
#include <string>
#include <vector>

#include "../../include/denseflow_b200.h"
#include "common.cuh"

namespace dfb {

struct LevelGeom {
    int w, h, pitch;
};

// set_param's value checks.  NaN fails every comparison and an infinity fails the range, so neither passes; a value that
// passes converts to int without loss.
inline bool whole_in(double v, double lo, double hi) { return v >= lo && v <= hi && v == std::floor(v); }
inline bool is_flag(double v) { return v == 0 || v == 1; }

// CUDA-event timing of an engine's dominant kernel: one event pair around each timed range of launches on one stream, read
// lazily so that timing never waits for the GPU inside a flow call.
class KernelTimer {
  public:
    KernelTimer() = default;
    KernelTimer(const KernelTimer &) = delete;
    KernelTimer &operator=(const KernelTimer &) = delete;
    ~KernelTimer() {
        for (auto &e : ev_)
            for (auto ev : e)
                if (ev) cudaEventDestroy(ev);
    }
    void begin(cudaStream_t s) {
        if (used_ == kRing) drain();
        if (!ev_[0][0])
            for (auto &e : ev_) {
                DFB_CUDA(cudaEventCreate(&e[0]));
                DFB_CUDA(cudaEventCreate(&e[1]));
            }
        DFB_CUDA(cudaEventRecord(ev_[used_][0], s));
    }
    // the range holds `launches` kernel launches and finishes `pairs` frame pairs
    void end(cudaStream_t s, uint64_t launches, uint64_t pairs) {
        DFB_CUDA(cudaEventRecord(ev_[used_][1], s));
        ++used_;
        launches_ += launches;
        pairs_ += pairs;
    }
    void read(uint64_t *launches, uint64_t *ns, uint64_t *pairs) {
        drain();
        *launches = launches_;
        *ns = ns_;
        *pairs = pairs_;
    }
    void reset() {
        drain();
        launches_ = ns_ = pairs_ = 0;
    }

  private:
    void drain() {
        for (int i = 0; i < used_; ++i) {
            DFB_CUDA(cudaEventSynchronize(ev_[i][1]));
            float ms = 0.f;
            DFB_CUDA(cudaEventElapsedTime(&ms, ev_[i][0], ev_[i][1]));
            ns_ += (uint64_t)((double)ms * 1e6);
        }
        used_ = 0;
    }
    static constexpr int kRing = 256;
    cudaEvent_t ev_[kRing][2] = {};
    int used_ = 0;
    uint64_t launches_ = 0, ns_ = 0, pairs_ = 0;
};

// Algorithm back-end working on device buffers. One frame "slot" holds everything that depends on
// a single frame (its fp32 pyramid), so a frame shared by two consecutive pairs is prepared once.
class FlowAlgorithm {
  public:
    virtual ~FlowAlgorithm() = default;
    virtual const char *name() const = 0;
    int num_slots() const { return (int)slots_.size(); }
    void ensure_slots(int n) {
        while ((int)slots_.size() < n) slots_.push_back(owned_zeroed(slot_elems_));
    }
    // per-frame work, u8 -> fp32 (+ pyramid), for n frames of one size and one row pitch at once (each launch of the per-frame
    // stages takes several frames: they are launch-latency-bound)
    virtual void prepare_frames(int n, const uint8_t *const *srcs, size_t pitch_bytes, int w, int h, const int *slots, cudaStream_t s) = 0;
    // per-pair work: flow(slot_a -> slot_b) of several independent pairs at once (the fused tvl1 engine runs them side by side
    // on disjoint SM groups)
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
        // fx set (bound = 0): the merge epilogue writes u1 to fx and u2 to fy as two float planes (row pitch f_pitch bytes), the
        // payloads of an h5 file's flow_x / flow_y datasets, INSTEAD of the float2 field; flow_xy may then be null
        float *fx = nullptr, *fy = nullptr;
        size_t f_pitch = 0;
        // init_x set (use_initial_flow): the solve starts from this flow instead of zero.  It is read before the pair's output
        // is written, so it may be the same memory.  Pixel (x, y) of the x channel is init_x[y * init_pitch + x * init_step] and
        // of the y channel init_y[...]: init_step 2 for a float2 field, 1 for two planes; init_pitch in floats.
        const float *init_x = nullptr, *init_y = nullptr;
        size_t init_pitch = 0;
        int init_step = 1;
    };
    virtual int max_concurrent_pairs(int w, int h) = 0;
    // after a CUDA error: what the engine's own watchdogs recorded (empty if nothing)
    virtual std::string fault_info() { return {}; }
    virtual void solve_batch(const PairJob *jobs, int n, int w, int h, cudaStream_t s) = 0;
    virtual bool set_param(const std::string &name, double v) = 0;
    virtual bool get_param(const std::string &name, double *v) const = 0;
    virtual void tvl1_stats(dfb_tvl1_stats *out) { *out = dfb_tvl1_stats{}; }
    // per-pair iteration logs of the most recent batch call: begin_batch() restarts the numbering
    virtual void begin_batch() {}
    virtual bool pair_stats(int pair_index, dfb_tvl1_stats *out) { (void)pair_index; *out = dfb_tvl1_stats{}; return false; }
    virtual void phase_ns(uint64_t *out) { for (int i = 0; i < 32; ++i) out[i] = 0; }
    virtual void reset_counters() {
        launches = 0;
        pixel_iters = 0;
        pixel_chunks = 0;
        timer_.reset();
    }
    void kernel_timing(uint64_t *launches_, uint64_t *ns, uint64_t *pairs) { timer_.read(launches_, ns, pairs); }
    // test hook behind dfb_debug_run_kernel: run one stage of this engine, through its own launch code and buffers, on dense
    // host planes (w x h floats each), with an optional scalar result.  Returns false when `kernel` is not one of the engine's stages.
    virtual bool debug_run(const std::string &kernel, const float *const *in, int n_in, float *const *out, int n_out, int w, int h,
                           const double *scalars, int n_scalars, double *scalar_out) {
        (void)kernel; (void)in; (void)n_in; (void)out; (void)n_out; (void)w; (void)h; (void)scalars; (void)n_scalars; (void)scalar_out;
        return false;
    }
    uint64_t launches = 0;     // kernels launched
    uint64_t pixel_iters = 0;  // tvl1: sum of level pixels over executed inner iterations
    uint64_t pixel_chunks = 0; // fused tvl1: sum of level pixels over tile visits (k iterations each)

  protected:
    static constexpr int kInitialSlots = 4;
    // the first kInitialSlots frame slots, `elems` floats each, come from the engine's slab; ensure_slots() adds owned ones
    void carve_slots(Slab &slab, size_t elems) {
        slot_elems_ = elems;
        for (int i = 0; i < kInitialSlots; ++i) slots_.push_back(slab.take<float>(elems));
    }
    // Device memory added after create time, freed with the engine.  It is zeroed because padding columns are read (never
    // used) by vectorised kernels.  The memset runs on the null stream, which the handle's non-blocking streams do not wait
    // for: finish it before any of them can touch the memory.
    float *owned_zeroed(size_t elems) {
        DeviceBuffer<float> &b = owned_.emplace_back();
        b.allocate(elems * sizeof(float));
        DFB_CUDA(cudaMemset(b, 0, b.bytes()));
        DFB_CUDA(cudaDeviceSynchronize());
        return b;
    }
    std::vector<float *> slots_;
    KernelTimer timer_;

  private:
    size_t slot_elems_ = 0;
    std::deque<DeviceBuffer<float>> owned_;
};

// Host-plane staging of the test hooks (debug_run, dfb_debug_run_kernel), on the null stream.  fill_plane sets every byte of
// the pitched plane p, padding and its spare row included; upload_rows (after fill_plane(p, fill) when fill >= 0) copies rows
// [row0, row0 + p.h) of a dense host plane p.w floats wide into p, and download_rows copies p back to the same rows.
inline void fill_plane(const Plane &p, int fill) { DFB_CUDA(cudaMemset(p.p, fill, (size_t)p.pitch * (p.h + 1) * sizeof(float))); }
inline void upload_rows(const Plane &p, const float *src, int row0, int fill = -1) {
    if (fill >= 0) fill_plane(p, fill);
    DFB_CUDA(cudaMemcpy2D(p.p, (size_t)p.pitch * 4, src + (size_t)row0 * p.w, (size_t)p.w * 4, (size_t)p.w * 4, p.h, cudaMemcpyHostToDevice));
}
inline void download_rows(float *dst, const Plane &p, int row0) {
    DFB_CUDA(cudaMemcpy2D(dst + (size_t)row0 * p.w, (size_t)p.w * 4, p.p, (size_t)p.pitch * 4, (size_t)p.w * 4, p.h, cudaMemcpyDeviceToHost));
}

// The start of a warm-started test pair as the flow calls pass one: rows [row0, row0 + h) of the dense host planes x, y (w
// floats wide), laid out in buf as a float2 field (step 2) or as two planes (step 1), rows `pitch` floats apart, with NaN in
// the padding.  Points pj's init_* fields at it.
inline void stage_initial_flow(DeviceBuffer<float> &buf, FlowAlgorithm::PairJob &pj, const float *x, const float *y, int row0, int w,
                               int h, int step, size_t pitch) {
    const size_t yoff = step == 2 ? 1 : pitch * h, elems = pitch * h * (step == 1 ? 2 : 1);
    std::vector<float> host(elems);
    std::memset(host.data(), 0xff, elems * sizeof(float));
    x += (size_t)row0 * w;
    y += (size_t)row0 * w;
    for (int r = 0; r < h; ++r)
        for (int c = 0; c < w; ++c) {
            host[r * pitch + (size_t)c * step] = x[(size_t)r * w + c];
            host[yoff + r * pitch + (size_t)c * step] = y[(size_t)r * w + c];
        }
    buf.allocate(elems * sizeof(float));
    DFB_CUDA(cudaMemcpy(buf, host.data(), elems * sizeof(float), cudaMemcpyHostToDevice));
    pj.init_x = buf;
    pj.init_y = buf + yoff;
    pj.init_pitch = pitch;
    pj.init_step = step;
}

std::unique_ptr<FlowAlgorithm> make_tvl1(int device, int max_w, int max_h);
std::unique_ptr<FlowAlgorithm> make_farneback(int device, int max_w, int max_h);

}  // namespace dfb
