// dfb_api.cu — the extern "C" boundary declared in include/denseflow_b200.h.
// Replaces the statements of the per-pair loop of DenseFlow::calc_optflows_imp
// (/root/reference/src/denseflow_gpu.cpp:313-342): upload x2 (:317-318), calc (:327/:329),
// download (:339) — plus the batch shape of the whole function (:307-342).
#include <cstdlib>
#include <type_traits>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "engine.h"
#include "jpeg.h"
#include "png_pack.h"
#include "preproc.h"
#include "tvl1.cuh"

using namespace dfb;

struct dfb_handle {
    int device = 0;
    int max_w = 0, max_h = 0;
    std::string algorithm;
    std::unique_ptr<FlowAlgorithm> alg;
    std::string last_error;
    dfb_counters counters{};

    // host-path plumbing: three streams so H2D of frame i+1, compute of pair i and D2H of flow i-1 overlap
    cudaStream_t s_in = nullptr, s_compute = nullptr, s_out = nullptr;
    static constexpr int kFrameRing = 16; // device u8 frames (dead as soon as their pyramid is built)
    static constexpr int kFlowRing = 128; // device flow / quantised outputs: two launches of up to 64 pairs in flight; slots are
                                          // allocated on first use and a call cycles through 2 x (pairs per launch) of them
    uint8_t *d_frame[kFrameRing] = {};
    size_t d_frame_pitch = 0;
    float *d_flow[kFlowRing] = {};
    uint8_t *d_qx[kFlowRing] = {}, *d_qy[kFlowRing] = {};
    cudaEvent_t ev_in[kFrameRing] = {}, ev_pyr[kFrameRing] = {}, ev_done[kFlowRing] = {}, ev_out[kFlowRing] = {};
    // pinned staging for pageable caller buffers
    uint8_t *h_frame[kFrameRing] = {};
    float *h_flow[kFlowRing] = {};
    uint8_t *h_q[kFlowRing] = {};
    std::unique_ptr<JpegEncoder> jpeg;  // nvJPEG encoder / decoder states, created on first use
    // scratch of dfb_process_bgr_batch_host (grown on demand)
    cudaStream_t s_fetch = nullptr;       // bitstream read-back of the BGR chain
    std::vector<cudaEvent_t> pb_events;   // events of the BGR chain (grown on demand)
    uint8_t *pb_bgr = nullptr, *pb_gray = nullptr, *pb_frames = nullptr, *pb_q = nullptr;
    size_t pb_bgr_cap = 0, pb_gray_cap = 0, pb_frames_cap = 0, pb_q_cap = 0;
    uint8_t *dec_bgr = nullptr;  // BGR scratch of dfb_decode_jpeg_gray_device
    size_t dec_bgr_cap = 0;
    void *png_scratch = nullptr;  // min/max partials + ticket + bounds of dfb_flow_to_png_image_device
    ResizeTap *d_taps = nullptr;  // resize coefficient tables on the device, rebuilt when the geometry changes
    int taps_cap = 0, taps_sw = 0, taps_sh = 0, taps_dw = 0, taps_dh = 0;
};

namespace {

std::mutex g_err_mutex;
std::string g_create_error;

int fail(dfb_handle *h, int code, const std::string &msg) {
    if (h)
        h->last_error = msg;
    else {
        std::lock_guard<std::mutex> lk(g_err_mutex);
        g_create_error = msg;
    }
    return code;
}

// after a failure in the middle of a call no copy into a caller buffer may still be in flight when the call returns
void quiesce(dfb_handle *h) {
    if (!h) return;
    for (cudaStream_t s : {h->s_in, h->s_compute, h->s_out, h->s_fetch})
        if (s) cudaStreamSynchronize(s);
    cudaGetLastError();
}

template <typename F> int guarded(dfb_handle *h, F &&f) {
    try {
        return f();
    } catch (const CudaError &e) {
        quiesce(h);
        std::string info;
        if (h && h->alg) info = h->alg->fault_info();
        return fail(h, DFB_ERR_CUDA, info.empty() ? std::string(e.what()) : std::string(e.what()) + " [" + info + "]");
    } catch (const std::exception &e) {
        quiesce(h);
        return fail(h, DFB_ERR_INVALID_ARG, e.what());
    } catch (...) {
        quiesce(h);
        return fail(h, DFB_ERR_INVALID_ARG, "unknown exception");
    }
}

// 1: page-locked (or managed) host memory the copy engines can reach directly; 0: pageable host memory (staged through
// the handle's pinned ring); -1: a device pointer, which the host entry points reject
int host_pointer_kind(const void *p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (a.type == cudaMemoryTypeDevice) return -1;
    return (a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged) ? 1 : 0;
}
bool is_pinned_host(const void *p) { return host_pointer_kind(p) == 1; }

int check_size(dfb_handle *h, int w, int h_) {
    if (w <= 0 || h_ <= 0) return fail(h, DFB_ERR_INVALID_ARG, "width/height must be positive");
    if (w > h->max_w || h_ > h->max_h)
        return fail(h, DFB_ERR_SIZE, "frame " + std::to_string(w) + "x" + std::to_string(h_) + " exceeds the " +
                                         std::to_string(h->max_w) + "x" + std::to_string(h->max_h) + " given to dfb_create");
    return DFB_OK;
}

// pinned staging buffers exist only for callers that pass pageable memory: allocated on first use
uint8_t *stage_frame(dfb_handle *h, int r) {
    if (!h->h_frame[r]) DFB_CUDA(cudaHostAlloc(&h->h_frame[r], (size_t)h->max_w * h->max_h, cudaHostAllocDefault));
    return h->h_frame[r];
}
float *stage_flow(dfb_handle *h, int r) {
    if (!h->h_flow[r]) DFB_CUDA(cudaHostAlloc(&h->h_flow[r], (size_t)h->max_w * h->max_h * 2 * sizeof(float), cudaHostAllocDefault));
    return h->h_flow[r];
}
uint8_t *stage_q(dfb_handle *h, int r) {
    if (!h->h_q[r]) DFB_CUDA(cudaHostAlloc(&h->h_q[r], (size_t)h->max_w * h->max_h * 2, cudaHostAllocDefault));
    return h->h_q[r];
}

void ensure_host_path(dfb_handle *h) {
    if (h->s_in) return;
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking));
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking));
    const size_t fpitch = (size_t)round_up(h->max_w, 128);
    h->d_frame_pitch = fpitch;
    for (int i = 0; i < dfb_handle::kFrameRing; ++i) {
        DFB_CUDA(cudaMalloc(&h->d_frame[i], fpitch * h->max_h));
        DFB_CUDA(cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming));
        DFB_CUDA(cudaEventCreateWithFlags(&h->ev_pyr[i], cudaEventDisableTiming));
    }
}

// output ring slots [0, n): allocated on first use (a 1080p handle runs 7 pairs per launch and touches 14 slots, a 340x256
// one up to 64 pairs per launch)
void ensure_flow_ring(dfb_handle *h, int n, bool quantised) {
    for (int i = 0; i < n; ++i) {
        if (!h->ev_done[i]) {
            DFB_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
            DFB_CUDA(cudaEventCreateWithFlags(&h->ev_out[i], cudaEventDisableTiming));
        }
        if (!quantised && !h->d_flow[i]) DFB_CUDA(cudaMalloc(&h->d_flow[i], (size_t)h->max_w * h->max_h * 2 * sizeof(float)));
        if (quantised && !h->d_qx[i]) {
            DFB_CUDA(cudaMalloc(&h->d_qx[i], (size_t)h->max_w * h->max_h));
            DFB_CUDA(cudaMalloc(&h->d_qy[i], (size_t)h->max_w * h->max_h));
        }
    }
}

// The batch shape of calc_optflows_imp (src/denseflow_gpu.cpp:307-342) over host buffers.
// quantise: bound > 0 => emit two u8 planes per pair instead of the float2 field.
int batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int w, int hh, float *const *flows,
               int bound, uint8_t *const *qx, uint8_t *const *qy) {
    if (int rc = check_size(h, w, hh)) return rc;
    if (n_frames < 0 || !frames) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    const int astep = std::abs(step);
    const int M = std::max(n_frames - astep, 0);  // :308
    if (M == 0) return DFB_OK;
    for (int f = 0; f < n_frames; ++f)
        if (!frames[f] || host_pointer_kind(frames[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "frames[" + std::to_string(f) + "] is null or a device pointer (host entry point: use dfb_calc_batch_device)");
    for (int j = 0; j < M; ++j) {
        const void *o0 = bound > 0 ? (const void *)qx[j] : (const void *)flows[j], *o1 = bound > 0 ? (const void *)qy[j] : o0;
        if (!o0 || !o1 || host_pointer_kind(o0) < 0 || host_pointer_kind(o1) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "output " + std::to_string(j) + " is null or a device pointer (host entry point)");
    }
    ensure_host_path(h);
    FlowAlgorithm &alg = *h->alg;
    alg.begin_batch();
    // pairs per solve_batch call; the frame slots hold one group plus the look-ahead frame
    const int B = std::max(1, std::min(alg.max_concurrent_pairs(w, hh), dfb_handle::kFlowRing / 2));
    alg.ensure_slots(B + astep + 1);
    const int nslots = alg.num_slots();
    const size_t fbytes = (size_t)w * hh;
    constexpr int FR = dfb_handle::kFrameRing;
    const int OR = 2 * B;  // two groups of pairs in flight
    // the unfused tvl1 schedule needs the float2 field as scratch even when only the quantised planes are wanted
    ensure_flow_ring(h, OR, bound > 0);
    double fused_flag = 1;
    if (bound > 0 && alg.get_param("fused", &fused_flag) && fused_flag == 0) ensure_flow_ring(h, OR, false);

    int uploaded = 0;  // frames [0, uploaded) have H2D + pyramid enqueued
    auto upload_until = [&](int last) {
        // sub-batches of at most FR frames: one H2D per frame on s_in, then ONE batched preparation on s_compute (the per-frame
        // stages are launch-latency-bound; a device ring slot is reused only after its frame has been prepared)
        while (uploaded <= last) {
            const int first = uploaded, cnt = std::min(last - uploaded + 1, FR);
            const uint8_t *srcs[FR];
            int slots[FR];
            for (int i = 0; i < cnt; ++i) {
                const int f = first + i, r = f % FR;
                if (f >= FR) DFB_CUDA(cudaStreamWaitEvent(h->s_in, h->ev_pyr[r], 0));  // ring slot's pyramid is built
                const uint8_t *src = frames[f];
                if (!is_pinned_host(src)) {
                    // the pinned staging buffer of this ring slot is free once its previous H2D finished
                    if (f >= FR) DFB_CUDA(cudaEventSynchronize(h->ev_in[r]));
                    std::memcpy(stage_frame(h, r), src, fbytes);
                    src = h->h_frame[r];
                }
                DFB_CUDA(cudaMemcpy2DAsync(h->d_frame[r], h->d_frame_pitch, src, w, w, hh, cudaMemcpyHostToDevice, h->s_in));
                DFB_CUDA(cudaEventRecord(h->ev_in[r], h->s_in));
                h->counters.h2d_bytes += fbytes;
                srcs[i] = h->d_frame[r];
                slots[i] = f % nslots;
            }
            DFB_CUDA(cudaStreamWaitEvent(h->s_compute, h->ev_in[(first + cnt - 1) % FR], 0));  // s_in is in order: the last covers all
            alg.prepare_frames(cnt, srcs, h->d_frame_pitch, w, hh, slots, h->s_compute);
            for (int i = 0; i < cnt; ++i) DFB_CUDA(cudaEventRecord(h->ev_pyr[(first + i) % FR], h->s_compute));
            uploaded += cnt;
        }
    };

    std::vector<int> pending_copy(OR, -1);  // pair index whose staged output still has to be memcpy'd out
    auto drain = [&](int ring) {
        const int j = pending_copy[ring];
        if (j < 0) return;
        DFB_CUDA(cudaEventSynchronize(h->ev_out[ring]));
        if (bound > 0) {
            std::memcpy(qx[j], h->h_q[ring], fbytes);
            std::memcpy(qy[j], h->h_q[ring] + fbytes, fbytes);
        } else {
            std::memcpy(flows[j], h->h_flow[ring], fbytes * 2 * sizeof(float));
        }
        pending_copy[ring] = -1;
    };

    std::vector<FlowAlgorithm::PairJob> jobs(B);
    for (int j0 = 0; j0 < M; j0 += B) {
        const int m = std::min(B, M - j0);
        // frames of this group (+ one ahead, so its H2D overlaps the solve)
        const int last_needed = j0 + m - 1 + astep;  // pairs j0..j0+m-1 touch frames j0..j0+m-1+|step| for either sign of step
        upload_until(std::min(last_needed + 1, n_frames - 1));
        for (int i = 0; i < m; ++i) {
            const int j = j0 + i;
            const int a = step > 0 ? j : j + astep;  // :315
            const int b = step > 0 ? j + astep : j;  // :316
            const int ring = j % OR;
            drain(ring);
            if (j >= OR) DFB_CUDA(cudaStreamWaitEvent(h->s_compute, h->ev_out[ring], 0));  // device output slot is free
            FlowAlgorithm::PairJob &pj = jobs[i];
            pj = FlowAlgorithm::PairJob{};
            pj.slot_a = a % nslots;
            pj.slot_b = b % nslots;
            pj.flow_xy = h->d_flow[ring];  // null in quantised mode unless the engine needs the scratch (see above)
            pj.flow_pitch_bytes = (size_t)w * 2 * sizeof(float);
            if (bound > 0) {  // f1: the engine's merge epilogue writes the two uint8 planes directly
                pj.bound = bound;
                pj.qx = h->d_qx[ring];
                pj.qy = h->d_qy[ring];
                pj.q_pitch = (size_t)w;
            }
        }
        alg.solve_batch(jobs.data(), m, w, hh, h->s_compute);
        DFB_CUDA(cudaEventRecord(h->ev_done[j0 % OR], h->s_compute));
        DFB_CUDA(cudaStreamWaitEvent(h->s_out, h->ev_done[j0 % OR], 0));
        for (int i = 0; i < m; ++i) {
            const int j = j0 + i, ring = j % OR;
            if (bound > 0) {
                const bool direct = is_pinned_host(qx[j]) && is_pinned_host(qy[j]);
                uint8_t *dx = direct ? qx[j] : stage_q(h, ring), *dy = direct ? qy[j] : stage_q(h, ring) + fbytes;
                DFB_CUDA(cudaMemcpyAsync(dx, h->d_qx[ring], fbytes, cudaMemcpyDeviceToHost, h->s_out));
                DFB_CUDA(cudaMemcpyAsync(dy, h->d_qy[ring], fbytes, cudaMemcpyDeviceToHost, h->s_out));
                if (!direct) pending_copy[ring] = j;
                h->counters.d2h_bytes += 2 * fbytes;
            } else {
                const bool direct = is_pinned_host(flows[j]);
                DFB_CUDA(cudaMemcpyAsync(direct ? flows[j] : stage_flow(h, ring), h->d_flow[ring], fbytes * 2 * sizeof(float),
                                         cudaMemcpyDeviceToHost, h->s_out));
                if (!direct) pending_copy[ring] = j;
                h->counters.d2h_bytes += fbytes * 2 * sizeof(float);
            }
            DFB_CUDA(cudaEventRecord(h->ev_out[ring], h->s_out));
            ++h->counters.pairs;  // total_flows += 1 (:340)
        }
    }
    DFB_CUDA(cudaStreamSynchronize(h->s_out));
    for (int r = 0; r < OR; ++r) drain(r);
    DFB_CUDA(cudaStreamSynchronize(h->s_compute));
    return DFB_OK;
}

}  // namespace

extern "C" {

const char *dfb_version(void) {
#ifdef DFB_STRICT_FP
    return "denseflow_b200 0.1 (sm_90a, strict-fp)";
#else
    return "denseflow_b200 0.1 (sm_90a)";
#endif
}

int dfb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int dfb_create(const char *algorithm, int device, int max_width, int max_height, dfb_handle **out) {
    if (!out) return fail(nullptr, DFB_ERR_INVALID_ARG, "out is null");
    *out = nullptr;
    if (!algorithm) return fail(nullptr, DFB_ERR_INVALID_ARG, "algorithm is null");
    const std::string alg(algorithm);
    if (alg == "nv") return fail(nullptr, DFB_ERR_UNSUPPORTED, "NV hardware flow not enabled, pls recompile");
    if (alg == "brox") return fail(nullptr, DFB_ERR_UNSUPPORTED, "brox is not supported in this build (tvl1 | farn)");
    if (alg != "tvl1" && alg != "farn") return fail(nullptr, DFB_ERR_UNKNOWN_ALGORITHM, "unknown optical algorithm " + alg);
    if (max_width <= 0 || max_height <= 0) return fail(nullptr, DFB_ERR_INVALID_ARG, "max_width/max_height must be positive");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(nullptr, DFB_ERR_NO_DEVICE, "no CUDA device available (the engine has no CPU path)");
    }
    if (device < 0 || device >= ndev) return fail(nullptr, DFB_ERR_INVALID_ARG, "device index out of range");
    dfb_handle *h = new dfb_handle();
    h->device = device;
    h->max_w = max_width;
    h->max_h = max_height;
    h->algorithm = alg;
    const int rc = guarded(nullptr, [&]() {
        DFB_CUDA(cudaSetDevice(device));
        h->alg = alg == "tvl1" ? make_tvl1(device, max_width, max_height) : make_farneback(device, max_width, max_height);
        return DFB_OK;
    });
    if (rc != DFB_OK) {
        delete h;
        return rc;
    }
    *out = h;
    return DFB_OK;
}

void dfb_destroy(dfb_handle *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < dfb_handle::kFrameRing; ++i) {
        if (h->d_frame[i]) cudaFree(h->d_frame[i]);
        if (h->h_frame[i]) cudaFreeHost(h->h_frame[i]);
        if (h->ev_in[i]) cudaEventDestroy(h->ev_in[i]);
        if (h->ev_pyr[i]) cudaEventDestroy(h->ev_pyr[i]);
    }
    for (int i = 0; i < dfb_handle::kFlowRing; ++i) {
        if (h->d_flow[i]) cudaFree(h->d_flow[i]);
        if (h->d_qx[i]) cudaFree(h->d_qx[i]);
        if (h->d_qy[i]) cudaFree(h->d_qy[i]);
        if (h->h_flow[i]) cudaFreeHost(h->h_flow[i]);
        if (h->h_q[i]) cudaFreeHost(h->h_q[i]);
        if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]);
        if (h->ev_out[i]) cudaEventDestroy(h->ev_out[i]);
    }
    h->jpeg.reset();
    for (void *p : {(void *)h->pb_bgr, (void *)h->pb_gray, (void *)h->pb_frames, (void *)h->pb_q})
        if (p) cudaFree(p);
    if (h->d_taps) cudaFree(h->d_taps);
    if (h->png_scratch) cudaFree(h->png_scratch);
    if (h->dec_bgr) cudaFree(h->dec_bgr);
    for (auto e : h->pb_events) cudaEventDestroy(e);
    if (h->s_fetch) cudaStreamDestroy(h->s_fetch);
    if (h->s_in) cudaStreamDestroy(h->s_in);
    if (h->s_compute) cudaStreamDestroy(h->s_compute);
    if (h->s_out) cudaStreamDestroy(h->s_out);
    h->alg.reset();
    delete h;
}

const char *dfb_last_error(const dfb_handle *h) {
    if (h) return h->last_error.c_str();
    std::lock_guard<std::mutex> lk(g_err_mutex);
    static thread_local std::string copy;
    copy = g_create_error;
    return copy.c_str();
}

int dfb_set_param(dfb_handle *h, const char *name, double value) {
    if (!h || !name) return DFB_ERR_INVALID_ARG;
    if (!h->alg->set_param(name, value)) return fail(h, DFB_ERR_INVALID_ARG, std::string("bad parameter ") + name);
    return DFB_OK;
}

int dfb_get_param(const dfb_handle *h, const char *name, double *value) {
    if (!h || !name || !value) return DFB_ERR_INVALID_ARG;
    return h->alg->get_param(name, value) ? DFB_OK : DFB_ERR_INVALID_ARG;
}

int dfb_calc_device(dfb_handle *h, const uint8_t *a, size_t a_pitch, const uint8_t *b, size_t b_pitch, int width,
                    int height, float *flow_xy, size_t flow_pitch, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!a || !b || !flow_xy) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (int rc = check_size(h, width, height)) return rc;
    if (a_pitch < (size_t)width || b_pitch < (size_t)width || flow_pitch < (size_t)width * 8)
        return fail(h, DFB_ERR_INVALID_ARG, "pitch smaller than a row");
    if ((reinterpret_cast<uintptr_t>(flow_xy) | flow_pitch) & 7)
        return fail(h, DFB_ERR_INVALID_ARG, "flow_xy and flow_pitch must be 8-byte aligned (CV_32FC2 rows)");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        h->alg->begin_batch();
        h->alg->prepare_frame(a, a_pitch, width, height, 0, s);
        h->alg->prepare_frame(b, b_pitch, width, height, 1, s);
        h->alg->solve(0, 1, width, height, flow_xy, flow_pitch, s);
        ++h->counters.pairs;
        return DFB_OK;
    });
}

int dfb_calc_host(dfb_handle *h, const uint8_t *a, const uint8_t *b, int width, int height, float *flow_xy) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!a || !b || !flow_xy) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    const uint8_t *frames[2] = {a, b};
    float *flows[1] = {flow_xy};
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        return batch_host(h, frames, 2, 1, width, height, flows, 0, nullptr, nullptr);
    });
}

int dfb_calc_batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                        float *const *flows) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (n_frames > std::abs(step) && !flows) return fail(h, DFB_ERR_INVALID_ARG, "flows is null");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        return batch_host(h, frames, n_frames, step, width, height, flows, 0, nullptr, nullptr);
    });
}

int dfb_calc_batch_host_u8(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                           int bound, uint8_t *const *qx, uint8_t *const *qy) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (bound <= 0) return fail(h, DFB_ERR_INVALID_ARG, "bound should > 0!");  // check_param, src/denseflow_gpu.cpp:15-18
    if (n_frames > std::abs(step) && (!qx || !qy)) return fail(h, DFB_ERR_INVALID_ARG, "qx/qy is null");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        return batch_host(h, frames, n_frames, step, width, height, nullptr, bound, qx, qy);
    });
}

int dfb_calc_batch_device(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                          float *flows, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (int rc = check_size(h, width, height)) return rc;
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    const int astep = std::abs(step);
    const int M = std::max(n_frames - astep, 0);
    if (M == 0) return DFB_OK;
    if (!frames || !flows) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        FlowAlgorithm &alg = *h->alg;
        alg.begin_batch();
        const int B = std::max(1, alg.max_concurrent_pairs(width, height));
        alg.ensure_slots(B + astep + 1);
        const int nslots = alg.num_slots();
        const size_t fbytes = (size_t)width * height;
        int prepared = 0;
        std::vector<FlowAlgorithm::PairJob> jobs(B);
        for (int j0 = 0; j0 < M; j0 += B) {
            const int m = std::min(B, M - j0);
            {
                std::vector<const uint8_t *> srcs;
                std::vector<int> slots;
                for (; prepared <= j0 + m - 1 + astep; ++prepared) {
                    srcs.push_back(frames + (size_t)prepared * fbytes);
                    slots.push_back(prepared % nslots);
                }
                if (!srcs.empty()) alg.prepare_frames((int)srcs.size(), srcs.data(), width, width, height, slots.data(), s);
            }
            for (int i = 0; i < m; ++i) {
                const int j = j0 + i;
                const int a = step > 0 ? j : j + astep;
                const int b = step > 0 ? j + astep : j;
                jobs[i] = FlowAlgorithm::PairJob{};
                jobs[i].slot_a = a % nslots;
                jobs[i].slot_b = b % nslots;
                jobs[i].flow_xy = flows + (size_t)j * fbytes * 2;
                jobs[i].flow_pitch_bytes = (size_t)width * 8;
            }
            alg.solve_batch(jobs.data(), m, width, height, s);
            h->counters.pairs += m;
        }
        return DFB_OK;
    });
}

int dfb_quantise_device(dfb_handle *h, const float *flow_xy, size_t flow_pitch, int width, int height, int bound,
                        uint8_t *qx, uint8_t *qy, size_t q_pitch, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!flow_xy || !qx || !qy) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (bound <= 0) return fail(h, DFB_ERR_INVALID_ARG, "bound should > 0!");
    if (width <= 0 || height <= 0) return fail(h, DFB_ERR_INVALID_ARG, "width/height must be positive");
    if (flow_pitch < (size_t)width * 8 || q_pitch < (size_t)width) return fail(h, DFB_ERR_INVALID_ARG, "pitch smaller than a row");
    if ((reinterpret_cast<uintptr_t>(flow_xy) | flow_pitch) & 7)
        return fail(h, DFB_ERR_INVALID_ARG, "flow_xy and flow_pitch must be 8-byte aligned (CV_32FC2 rows)");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        launch_quantise(flow_xy, flow_pitch, width, height, bound, qx, qy, q_pitch, static_cast<cudaStream_t>(stream));
        ++h->alg->launches;
        return DFB_OK;
    });
}

int dfb_flow_to_png_image_device(dfb_handle *h, const float *flow_xy, size_t flow_pitch, int width, int height, uint8_t *bgr,
                                  size_t bgr_pitch, double *bounds_xy_host, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!flow_xy || !bgr) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (width <= 0 || height <= 0 || flow_pitch < (size_t)width * 8 || bgr_pitch < (size_t)width * 3)
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    if ((reinterpret_cast<uintptr_t>(flow_xy) | flow_pitch) & 7)
        return fail(h, DFB_ERR_INVALID_ARG, "flow_xy and flow_pitch must be 8-byte aligned (CV_32FC2 rows)");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (!h->png_scratch) {
            DFB_CUDA(cudaMalloc(&h->png_scratch, png_pack_scratch_bytes()));
            DFB_CUDA(cudaMemset(h->png_scratch, 0, png_pack_scratch_bytes()));
            DFB_CUDA(cudaDeviceSynchronize());
        }
        PngBounds *bd = nullptr;
        launch_flow_to_png_image(flow_xy, flow_pitch, width, height, bgr, bgr_pitch, h->png_scratch, &bd, s);
        h->alg->launches += 2;
        if (bounds_xy_host) {  // the caller wants the two bounds now: a blocking read-back of 16 bytes
            PngBounds b{};
            DFB_CUDA(cudaMemcpyAsync(&b, bd, sizeof(b), cudaMemcpyDeviceToHost, s));
            DFB_CUDA(cudaStreamSynchronize(s));
            bounds_xy_host[0] = b.bound_x;
            bounds_xy_host[1] = b.bound_y;
        }
        return DFB_OK;
    });
}

int dfb_bgr_to_gray_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int width, int height, uint8_t *gray,
                           size_t gray_pitch, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || !gray) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (width <= 0 || height <= 0 || bgr_pitch < (size_t)width * 3 || gray_pitch < (size_t)width)
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        launch_bgr_to_gray(bgr, bgr_pitch, width, height, gray, gray_pitch, static_cast<cudaStream_t>(stream));
        ++h->alg->launches;
        return DFB_OK;
    });
}

int dfb_resize_gray_device(dfb_handle *h, const uint8_t *src, size_t src_pitch, int sw, int sh, uint8_t *dst, size_t dst_pitch,
                           int dw, int dh, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!src || !dst) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0 || src_pitch < (size_t)sw || dst_pitch < (size_t)dw)
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (sw == dw && sh == dh) {  // cv::resize with an equal size is a copy
            DFB_CUDA(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, sw, sh, cudaMemcpyDeviceToDevice, s));
            return DFB_OK;
        }
        if (h->taps_sw != sw || h->taps_sh != sh || h->taps_dw != dw || h->taps_dh != dh) {
            std::vector<ResizeTap> xt, yt;
            build_resize_taps(dw, sw, true, xt);
            build_resize_taps(dh, sh, false, yt);
            if (dw + dh > h->taps_cap) {
                DFB_CUDA(cudaDeviceSynchronize());
                if (h->d_taps) DFB_CUDA(cudaFree(h->d_taps));
                h->taps_cap = dw + dh;
                DFB_CUDA(cudaMalloc(&h->d_taps, sizeof(ResizeTap) * h->taps_cap));
            } else {
                DFB_CUDA(cudaDeviceSynchronize());  // a launch with the old tables may still be running
            }
            DFB_CUDA(cudaMemcpy(h->d_taps, xt.data(), sizeof(ResizeTap) * dw, cudaMemcpyHostToDevice));
            DFB_CUDA(cudaMemcpy(h->d_taps + dw, yt.data(), sizeof(ResizeTap) * dh, cudaMemcpyHostToDevice));
            h->taps_sw = sw;
            h->taps_sh = sh;
            h->taps_dw = dw;
            h->taps_dh = dh;
        }
        launch_resize_u8(src, src_pitch, sw, sh, dst, dst_pitch, dw, dh, h->d_taps, h->d_taps + dw, s);
        ++h->alg->launches;
        return DFB_OK;
    });
}

size_t dfb_jpeg_max_bytes(int width, int height) {
    if (width <= 0 || height <= 0) return 0;
    return (size_t)width * height * 2 + 4096;  // far above any baseline gray JPEG of this size
}

int dfb_encode_jpeg_gray_device(dfb_handle *h, const uint8_t *gray, size_t gray_pitch, int width, int height, int quality,
                                uint8_t *out, size_t out_capacity, size_t *out_len, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!gray || !out || !out_len) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (width <= 0 || height <= 0 || gray_pitch < (size_t)width || quality < 1 || quality > 100)
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry or quality");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        if (!h->jpeg) h->jpeg.reset(new JpegEncoder());
        *out_len = h->jpeg->encode_gray(gray, gray_pitch, width, height, quality, out, out_capacity, static_cast<cudaStream_t>(stream));
        return DFB_OK;
    });
}

int dfb_decode_jpeg_gray_device(dfb_handle *h, const uint8_t *jpeg, size_t jpeg_len, uint8_t *gray, size_t gray_pitch, int max_width,
                                int max_height, int *width, int *height, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!jpeg || !jpeg_len || !gray || !width || !height) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (!h->jpeg) h->jpeg.reset(new JpegEncoder());
        int w = 0, hh = 0, nc = 0;
        h->jpeg->image_info(jpeg, jpeg_len, &w, &hh, &nc);
        *width = w;
        *height = hh;
        if (w <= 0 || hh <= 0) return fail(h, DFB_ERR_INVALID_ARG, "not a JPEG image");
        if (w > max_width || hh > max_height || gray_pitch < (size_t)w)
            return fail(h, DFB_ERR_SIZE, "decoded frame " + std::to_string(w) + "x" + std::to_string(hh) + " does not fit the output buffer");
        const size_t need = (size_t)w * hh * 3;
        if (need > h->dec_bgr_cap) {
            DFB_CUDA(cudaDeviceSynchronize());
            if (h->dec_bgr) DFB_CUDA(cudaFree(h->dec_bgr));
            DFB_CUDA(cudaMalloc(&h->dec_bgr, need));
            h->dec_bgr_cap = need;
        }
        // imread(IMREAD_COLOR) -> BGR, then the decode stage's cvtColor(BGR2GRAY) (src/denseflow_gpu.cpp:160-163), bit-exact from there on
        h->jpeg->decode_bgr(jpeg, jpeg_len, h->dec_bgr, (size_t)w * 3, w, hh, s);
        launch_bgr_to_gray(h->dec_bgr, (size_t)w * 3, w, hh, gray, gray_pitch, s);
        ++h->alg->launches;
        return (int)DFB_OK;
    });
}

int dfb_process_bgr_batch_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int sw, int sh, int dw, int dh,
                               int bound, int jpeg_quality, uint8_t *const *jpg_x, uint8_t *const *jpg_y, size_t capacity,
                               size_t *len_x, size_t *len_y) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || n_frames < 0) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    if (bound <= 0) return fail(h, DFB_ERR_INVALID_ARG, "bound should > 0!");
    if (sw <= 0 || sh <= 0 || dw < 0 || dh < 0 || (dw == 0) != (dh == 0)) return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    if (dw == 0) {
        dw = sw;
        dh = sh;
    }
    if (int rc = check_size(h, dw, dh)) return rc;
    const int astep = std::abs(step);
    const int M = std::max(n_frames - astep, 0);
    if (M == 0) return DFB_OK;
    if (!jpg_x || !jpg_y || !len_x || !len_y) return fail(h, DFB_ERR_INVALID_ARG, "null output");
    for (int f = 0; f < n_frames; ++f)
        if (!bgr[f] || host_pointer_kind(bgr[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "bgr[" + std::to_string(f) + "] is null or a device pointer (host entry point)");
    for (int j = 0; j < M; ++j)
        if (!jpg_x[j] || !jpg_y[j] || host_pointer_kind(jpg_x[j]) < 0 || host_pointer_kind(jpg_y[j]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "jpeg output " + std::to_string(j) + " is null or a device pointer (host entry point)");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        ensure_host_path(h);
        if (!h->s_fetch) DFB_CUDA(cudaStreamCreateWithFlags(&h->s_fetch, cudaStreamNonBlocking));
        FlowAlgorithm &alg = *h->alg;
        alg.begin_batch();
        auto grow = [&](auto *&ptr, size_t &cap, size_t need) {
            if (need <= cap) return;
            DFB_CUDA(cudaDeviceSynchronize());
            if (ptr) DFB_CUDA(cudaFree(ptr));
            void *p = nullptr;
            DFB_CUDA(cudaMalloc(&p, need));
            ptr = static_cast<std::remove_reference_t<decltype(ptr)>>(p);
            cap = need;
        };
        // Three stages on three streams, groups of B pairs in flight (the reference runs the same three stages as three host
        // threads around queues, include/dense_flow.h:76-80):
        //   s_in      H2D of BGR frame f -> cvtColor -> resize into the gray frame array        (decode stage tail, :163-170)
        //   s_compute pyramids / polynomial expansions + flow of group g, quantised planes out   (:313-342 + src/common.cpp:4-16)
        //   s_out     two JPEG encodes per pair of group g (nvJPEG, one encoder state per plane)  (src/common.cpp:56-57)
        //   s_fetch   bitstreams of group g-1 to the host while the GPU works on group g
        const int B = std::max(1, std::min(alg.max_concurrent_pairs(dw, dh), 8));
        const size_t fpx = (size_t)dw * dh, bgr_bytes = (size_t)sw * sh * 3;
        grow(h->pb_bgr, h->pb_bgr_cap, 2 * bgr_bytes);           // two staging frames: H2D of f+1 overlaps gray/resize of f
        grow(h->pb_gray, h->pb_gray_cap, (size_t)sw * sh);
        grow(h->pb_frames, h->pb_frames_cap, fpx * n_frames);
        grow(h->pb_q, h->pb_q_cap, fpx * 2 * 2 * B);              // quantised planes of two groups
        alg.ensure_slots(B + astep + 1);
        const int nslots = alg.num_slots();
        while ((int)h->pb_events.size() < n_frames + 8) {
            cudaEvent_t e;
            DFB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            h->pb_events.push_back(e);
        }
        cudaEvent_t *ev_frame = h->pb_events.data() + 8;          // [n_frames]
        cudaEvent_t *ev_gray = h->pb_events.data();                // [2] staging buffer consumed
        cudaEvent_t *ev_flow = h->pb_events.data() + 2;            // [2] group's planes ready
        cudaEvent_t *ev_enc = h->pb_events.data() + 4;             // [2] group's encodes done
        if (!h->jpeg) h->jpeg.reset(new JpegEncoder());
        h->jpeg->ensure_states(4 * B);

        int uploaded = 0;
        auto upload_until = [&](int last) {
            for (; uploaded <= std::min(last, n_frames - 1); ++uploaded) {
                const int f = uploaded, sb = f & 1;
                if (f >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_in, ev_gray[sb], 0));
                uint8_t *stage = h->pb_bgr + (size_t)sb * bgr_bytes;
                DFB_CUDA(cudaMemcpyAsync(stage, bgr[f], bgr_bytes, cudaMemcpyHostToDevice, h->s_in));
                h->counters.h2d_bytes += bgr_bytes;
                uint8_t *dst = h->pb_frames + fpx * f;
                if (dw == sw && dh == sh) {
                    launch_bgr_to_gray(stage, (size_t)sw * 3, sw, sh, dst, dw, h->s_in);
                } else {
                    launch_bgr_to_gray(stage, (size_t)sw * 3, sw, sh, h->pb_gray, sw, h->s_in);
                    const int rc = dfb_resize_gray_device(h, h->pb_gray, sw, sw, sh, dst, dw, dw, dh, h->s_in);
                    if (rc != DFB_OK) throw std::runtime_error(h->last_error);
                }
                alg.launches += 1;
                DFB_CUDA(cudaEventRecord(ev_gray[sb], h->s_in));
                DFB_CUDA(cudaEventRecord(ev_frame[f], h->s_in));
            }
        };
        int prepared = 0;
        std::vector<FlowAlgorithm::PairJob> jobs(B);
        auto flow_group = [&](int g) {
            const int j0 = g * B, m = std::min(B, M - j0), slot = g & 1;
            const int last_frame = j0 + m - 1 + astep;
            upload_until(last_frame + 1);
            DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev_frame[last_frame], 0));
            if (g >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev_enc[slot], 0));  // the planes of group g-2 have been encoded
            {
                std::vector<const uint8_t *> srcs;
                std::vector<int> slots;
                for (; prepared <= last_frame; ++prepared) {
                    srcs.push_back(h->pb_frames + fpx * prepared);
                    slots.push_back(prepared % nslots);
                }
                if (!srcs.empty()) alg.prepare_frames((int)srcs.size(), srcs.data(), dw, dw, dh, slots.data(), h->s_compute);
            }
            for (int i = 0; i < m; ++i) {
                const int j = j0 + i;
                FlowAlgorithm::PairJob &pj = jobs[i];
                pj = FlowAlgorithm::PairJob{};
                pj.slot_a = (step > 0 ? j : j + astep) % nslots;  // :315
                pj.slot_b = (step > 0 ? j + astep : j) % nslots;  // :316
                pj.bound = bound;
                pj.qx = h->pb_q + ((size_t)(slot * B + i) * 2) * fpx;
                pj.qy = pj.qx + fpx;
                pj.q_pitch = (size_t)dw;
            }
            alg.solve_batch(jobs.data(), m, dw, dh, h->s_compute);
            DFB_CUDA(cudaEventRecord(ev_flow[slot], h->s_compute));
            // encode stage (src/common.cpp:48-64): one JPEG per plane
            DFB_CUDA(cudaStreamWaitEvent(h->s_out, ev_flow[slot], 0));
            for (int i = 0; i < m; ++i) {
                const uint8_t *qx = h->pb_q + ((size_t)(slot * B + i) * 2) * fpx;
                h->jpeg->enqueue((slot * B + i) * 2, qx, dw, dw, dh, jpeg_quality, h->s_out);
                h->jpeg->enqueue((slot * B + i) * 2 + 1, qx + fpx, dw, dw, dh, jpeg_quality, h->s_out);
            }
            DFB_CUDA(cudaEventRecord(ev_enc[slot], h->s_out));
            h->counters.pairs += m;
        };
        auto finish_group = [&](int g) {
            const int j0 = g * B, m = std::min(B, M - j0), slot = g & 1;
            DFB_CUDA(cudaEventSynchronize(ev_enc[slot]));
            for (int i = 0; i < m; ++i)
                for (int c = 0; c < 2; ++c) {
                    const int st = (slot * B + i) * 2 + c;
                    const size_t len = h->jpeg->length(st, h->s_fetch);
                    if (len > capacity) throw std::runtime_error("jpeg output buffer too small (" + std::to_string(len) + " > " + std::to_string(capacity) + ")");
                    (c ? len_y : len_x)[j0 + i] = len;
                    h->jpeg->fetch(st, (c ? jpg_y : jpg_x)[j0 + i], len, h->s_fetch);
                    h->counters.d2h_bytes += len;
                }
            DFB_CUDA(cudaStreamSynchronize(h->s_fetch));
        };
        const int G = (M + B - 1) / B;
        for (int g = 0; g < G; ++g) {
            flow_group(g);
            if (g > 0) finish_group(g - 1);
        }
        finish_group(G - 1);
        DFB_CUDA(cudaStreamSynchronize(h->s_in));
        DFB_CUDA(cudaStreamSynchronize(h->s_compute));
        DFB_CUDA(cudaStreamSynchronize(h->s_out));
        return DFB_OK;
    });
}

int dfb_debug_run_kernel(dfb_handle *h, const char *kernel, const float *const *in, int n_in, float *const *out, int n_out, int width,
                         int height, const double *scalars, int n_scalars, double *scalars_out) {
    if (!h || !kernel) return DFB_ERR_INVALID_ARG;
    if (width <= 0 || height <= 0 || n_in < 0 || n_out < 0 || n_in > 16 || n_out > 16) return fail(h, DFB_ERR_INVALID_ARG, "bad arguments");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        const std::string k(kernel);
        if (h->alg->debug_run(k, in, n_in, out, n_out, width, height, scalars, n_scalars)) return DFB_OK;  // the engine's own stages
        auto sc = [&](int i) { return i < n_scalars ? scalars[i] : 0.0; };
        int ow = width, oh = height;
        if (k == "resize") {
            ow = (int)sc(0);
            oh = (int)sc(1);
            if (ow <= 0 || oh <= 0) throw std::runtime_error("resize: bad destination size");
        }
        const int pitch = round_up(width, 32), opitch = round_up(ow, 32);
        std::vector<float *> dev;
        auto alloc = [&](int w_, int h_, int p_) {
            float *p = nullptr;
            DFB_CUDA(cudaMalloc(&p, (size_t)p_ * (h_ + 1) * sizeof(float)));
            DFB_CUDA(cudaMemset(p, 0, (size_t)p_ * (h_ + 1) * sizeof(float)));
            dev.push_back(p);
            return Plane{p, w_, h_, p_};
        };
        std::vector<Plane> pin, pout;
        for (int i = 0; i < n_in; ++i) {
            pin.push_back(alloc(width, height, pitch));
            DFB_CUDA(cudaMemcpy2D(pin[i].p, (size_t)pitch * 4, in[i], (size_t)width * 4, (size_t)width * 4, height, cudaMemcpyHostToDevice));
        }
        double *d_part = nullptr, *d_sum = nullptr;
        auto need = [&](int ni, int no) {
            if (n_in != ni || n_out != no) throw std::runtime_error(k + ": expects " + std::to_string(ni) + " inputs and " + std::to_string(no) + " outputs");
        };
        int inplace_from = -1;  // outputs that are in-place updates of inputs starting at this input index
        if (k == "gradient") {
            need(1, 2);
            pout = {alloc(width, height, pitch), alloc(width, height, pitch)};
            launch_centered_gradient(pin[0], pout[0], pout[1], nullptr);
        } else if (k == "warp") {
            need(6, 4);
            for (int i = 0; i < 4; ++i) pout.push_back(alloc(width, height, pitch));
            launch_warp_backward(pin[0], pin[1], pin[2], pin[3], pin[4], pin[5], pout[0], pout[1], pout[2], pout[3], nullptr);
        } else if (k == "estimate_u") {
            need(10, 2);
            const Tvl1Consts c{(float)sc(0), 0.f, (float)sc(1)};
            const bool calc = sc(2) != 0;
            const int nblk = estimate_u_blocks(width, height);
            if (calc) {
                DFB_CUDA(cudaMalloc(&d_part, sizeof(double) * nblk));
                DFB_CUDA(cudaMalloc(&d_sum, sizeof(double)));
            }
            launch_estimate_u(pin[0], pin[1], pin[2], pin[3], pin[4], pin[5], pin[6], pin[7], pin[8], pin[9], c, d_part, nullptr);
            if (calc) {
                launch_sum_partials(d_part, nblk, d_sum, nullptr);
                if (scalars_out) DFB_CUDA(cudaMemcpy(scalars_out, d_sum, sizeof(double), cudaMemcpyDeviceToHost));
            }
            inplace_from = 8;
        } else if (k == "estimate_dual") {
            need(6, 4);
            const Tvl1Consts c{0.f, (float)sc(0), 0.f};
            launch_estimate_dual(pin[0], pin[1], pin[2], pin[3], pin[4], pin[5], c, nullptr);
            inplace_from = 2;
        } else if (k == "resize") {
            need(1, 1);
            pout = {alloc(ow, oh, opitch)};
            launch_resize_linear(pin[0], pout[0], (float)sc(2), (float)sc(3), n_scalars > 4 ? (float)sc(4) : 1.0f, nullptr);
        } else {
            for (float *p : dev) cudaFree(p);
            throw std::runtime_error("unknown debug kernel " + k);
        }
        DFB_CUDA(cudaDeviceSynchronize());
        for (int i = 0; i < n_out; ++i) {
            const Plane &src = inplace_from >= 0 ? pin[inplace_from + i] : pout[i];
            DFB_CUDA(cudaMemcpy2D(out[i], (size_t)src.w * 4, src.p, (size_t)src.pitch * 4, (size_t)src.w * 4, src.h, cudaMemcpyDeviceToHost));
        }
        for (float *p : dev) cudaFree(p);
        if (d_part) cudaFree(d_part);
        if (d_sum) cudaFree(d_sum);
        return DFB_OK;
    });
}

int dfb_debug_time_kernel(dfb_handle *h, const char *kernel, int width, int height, int sets, int reps, double *ms_per_launch) {
    if (!h || !kernel || !ms_per_launch) return DFB_ERR_INVALID_ARG;
    if (width <= 0 || height <= 0 || sets < 1 || sets > 64 || reps < 1) return fail(h, DFB_ERR_INVALID_ARG, "bad arguments");
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        const std::string k(kernel);
        const bool primal = k == "estimate_u";
        if (!primal && k != "estimate_dual") throw std::runtime_error("unknown kernel " + k);
        const int nplanes = primal ? 10 : 6;
        const int pitch = round_up(width, 32);
        const size_t pe = (size_t)pitch * (height + 1);
        float *buf = nullptr;
        DFB_CUDA(cudaMalloc(&buf, pe * sizeof(float) * nplanes * sets));
        auto plane = [&](int set, int i) { return Plane{buf + ((size_t)set * nplanes + i) * pe, width, height, pitch}; };
        for (int sidx = 0; sidx < sets; ++sidx)
            for (int i = 0; i < nplanes; ++i) launch_fill(plane(sidx, i), 0.125f * (float)(i + 1), nullptr);
        const Tvl1Consts c{0.045f, 0.25f / 0.3f, 0.3f};
        auto run = [&](int sidx) {
            if (primal)
                launch_estimate_u(plane(sidx, 0), plane(sidx, 1), plane(sidx, 2), plane(sidx, 3), plane(sidx, 4), plane(sidx, 5), plane(sidx, 6),
                                  plane(sidx, 7), plane(sidx, 8), plane(sidx, 9), c, nullptr, nullptr);
            else
                launch_estimate_dual(plane(sidx, 0), plane(sidx, 1), plane(sidx, 2), plane(sidx, 3), plane(sidx, 4), plane(sidx, 5), c, nullptr);
        };
        for (int i = 0; i < 3; ++i) run(i % sets);
        cudaEvent_t e0, e1;
        DFB_CUDA(cudaEventCreate(&e0));
        DFB_CUDA(cudaEventCreate(&e1));
        DFB_CUDA(cudaEventRecord(e0, nullptr));
        for (int i = 0; i < reps; ++i) run((i + 3) % sets);
        DFB_CUDA(cudaEventRecord(e1, nullptr));
        DFB_CUDA(cudaEventSynchronize(e1));
        float ms = 0.f;
        DFB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        *ms_per_launch = (double)ms / reps;
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        cudaFree(buf);
        return DFB_OK;
    });
}

int dfb_get_tvl1_stats(dfb_handle *h, dfb_tvl1_stats *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        h->alg->tvl1_stats(out);
        return DFB_OK;
    });
}

int dfb_get_tvl1_pair_stats(dfb_handle *h, int pair_index, dfb_tvl1_stats *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        if (!h->alg->pair_stats(pair_index, out)) return fail(h, DFB_ERR_INVALID_ARG, "pair_index is not one of the last 256 pairs of the most recent tvl1 batch call");
        return (int)DFB_OK;
    });
}

int dfb_get_counters(dfb_handle *h, dfb_counters *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        dfb_tvl1_stats st;
        h->alg->tvl1_stats(&st);  // folds a pending fused-kernel log into pixel_iters
        *out = h->counters;
        out->kernel_launches = h->alg->launches;
        out->pixel_iters = h->alg->pixel_iters;
        out->pixel_chunks = h->alg->pixel_chunks;
        h->alg->kernel_timing(&out->timed_kernel_launches, &out->timed_kernel_ns, &out->timed_kernel_pairs);
        return DFB_OK;
    });
}

int dfb_get_tvl1_phase_ns(dfb_handle *h, uint64_t out[32]) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        DFB_CUDA(cudaSetDevice(h->device));
        h->alg->phase_ns(out);
        return DFB_OK;
    });
}

int dfb_reset_counters(dfb_handle *h) {
    if (!h) return DFB_ERR_INVALID_ARG;
    h->counters = dfb_counters{};
    cudaSetDevice(h->device);
    h->alg->reset_counters();
    return DFB_OK;
}

}  // extern "C"
