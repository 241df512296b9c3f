// dfb_api.cu — the extern "C" boundary declared in include/denseflow_b200.h.
// Replaces the statements of the per-pair loop of DenseFlow::calc_optflows_imp
// (/root/reference/src/denseflow_gpu.cpp:313-342): upload x2 (:317-318), calc (:327/:329),
// download (:339) — plus the batch shape of the whole function (:307-342).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "engine.h"
#include "jpeg.h"
#include "jpeg_decode.h"
#include "jpeg_encode.h"
#include "png_encode.h"
#include "png_pack.h"
#include "preproc.h"
#include "tvl1.cuh"

using namespace dfb;

// resize coefficient tables on the device, rebuilt when the geometry changes
struct TapTable {
    DeviceBuffer<ResizeTap> d;
    int sw = 0, sh = 0, dw = 0, dh = 0;
};

// CUDA events created on first use and destroyed with their owner; they record no time unless flags says so
class Events {
  public:
    explicit Events(unsigned flags = cudaEventDisableTiming) : flags_(flags) {}
    Events(const Events &) = delete;
    Events &operator=(const Events &) = delete;
    ~Events() {
        for (cudaEvent_t e : e_) cudaEventDestroy(e);
    }
    void ensure(size_t n) {
        while (e_.size() < n) {
            cudaEvent_t e;
            DFB_CUDA(cudaEventCreateWithFlags(&e, flags_));
            e_.push_back(e);
        }
    }
    cudaEvent_t operator[](size_t i) const { return e_[i]; }

  private:
    unsigned flags_;
    std::vector<cudaEvent_t> e_;
};

struct dfb_handle {
    int device = 0;
    int max_w = 0, max_h = 0;
    std::string algorithm;
    std::unique_ptr<FlowAlgorithm> alg;
    std::string last_error;
    dfb_counters counters{};

    // host-path plumbing: three streams so H2D of frame i+1, compute of pair i and D2H of flow i-1 overlap
    cudaStream_t s_in = nullptr, s_compute = nullptr, s_out = nullptr;
    cudaStream_t s_fetch = nullptr;  // file read-back of the encoding pipelines
    static constexpr int kFrameRing = 16; // device u8 frames (dead as soon as their pyramid is built)
    static constexpr int kMaxGroup = 64;  // pairs per group of the calc calls; two groups are in flight
    DeviceBuffer<uint8_t> d_frame[kFrameRing];
    size_t d_frame_pitch = 0;
    Events ev_in, ev_pyr;     // [kFrameRing] frame uploaded, its pyramid built
    // pinned staging for pageable caller buffers (outputs: one per pair of the two groups in flight)
    PinnedBuffer<uint8_t> h_frame[kFrameRing];
    PinnedBuffer<uint8_t> h_out[2 * kMaxGroup];
    // the flow group loop (flow_groups): device outputs of two slots of B pairs, grown on demand, and per slot the events
    // that hand a solved group from s_compute to s_out and mark the slot free once its outputs are read back or encoded
    DeviceBuffer<uint8_t> flow_out;
    struct {
        Events solved, freed;  // [2]
    } flow_ev;
    std::unique_ptr<JpegEncoder> jpeg;  // nvJPEG encoder / decoder states, created on first use
    // scratch of the flow chains (dfb_process_*_batch_host), grown on demand
    DeviceBuffer<uint8_t> pb_bgr, pb_gray, pb_frames;
    struct {
        Events frame;      // [n_frames] frame f is in pb_frames
        Events gray;       // [2] BGR staging buffer consumed
    } chain_ev;
    DeviceBuffer<uint8_t> dec_bgr;      // BGR scratch of dfb_decode_jpeg_gray_device
    std::unique_ptr<JpegDecoder> jdec;  // imdecode-exact JPEG decoder, created on first use
    DeviceBuffer<uint8_t> png_scratch;  // min/max partials + ticket + bounds of dfb_flow_to_png_image_device
    std::unique_ptr<PngEncoder> png;    // imencode(".png") workspace and files, created on first use
    DeviceBuffer<uint8_t> png_bgr;      // packed images of the -st=png flow output, one per pair of its two slots
    TapTable gray_taps;  // dfb_resize_gray_device
    // scratch of the frame-extraction calls (-s=0), grown on demand
    TapTable ycc_taps;                // colour resize of all three calls
    DeviceBuffer<uint8_t> enc_ycc;    // Y / Cb / Cr planes of dfb_encode_jpeg_bgr_device
    DeviceBuffer<uint8_t> enc_gray;   // the block-padded copy of the plane dfb_encode_jpeg_gray_device hands nvJPEG
    DeviceBuffer<uint8_t> ex_bgr, ex_ycc;  // the -s=0 pipeline: BGR staging of its frame source, planes of two groups
    struct {
        Events h2d, conv;     // [2] BGR staging filled; the BGR source's staging frame consumed
        Events planes, enc;   // [2] a group's planes ready, its encodes done
    } extract_ev;
    // "jpeg_exact" = 1: every JPEG this handle writes is imencode(".jpg")'s bytes (JpegExactEncoder) instead of nvJPEG's
    bool jpeg_exact = false;
    std::unique_ptr<JpegExactEncoder> jex;  // created on first use

    ~dfb_handle() {
        for (cudaStream_t s : {s_in, s_compute, s_out, s_fetch})
            if (s) cudaStreamDestroy(s);
    }
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

}  // namespace

int dfb::fail_unbound(int code, const std::string &msg) { return fail(nullptr, code, msg); }

namespace {

// after a failure in the middle of a call no copy into a caller buffer may still be in flight when the call returns
void quiesce(dfb_handle *h) {
    if (!h) return;
    for (cudaStream_t s : {h->s_in, h->s_compute, h->s_out, h->s_fetch})
        if (s) cudaStreamSynchronize(s);
    cudaGetLastError();
}

// Runs f on the handle's device (h non-null); a CUDA error or an exception becomes the call's error code and message.
template <typename F> int guarded(dfb_handle *h, F &&f) {
    try {
        if (h) DFB_CUDA(cudaSetDevice(h->device));
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

// use_initial_flow = 1 on the handle: the calls with a float flow buffer read each pair's initial flow from it
bool initial_flow(const dfb_handle *h) {
    double v = 0;
    return h->alg->get_param("use_initial_flow", &v) && v != 0;
}
// a missing flow buffer; with use_initial_flow set it is also the missing input
int null_flow(dfb_handle *h, const std::string &what) {
    return fail(h, DFB_ERR_INVALID_ARG, initial_flow(h) ? what + ": use_initial_flow is set, so the flow buffer must hold the initial flow" : what);
}
// Where the outputs of a host flow call go.  Pair j has k buffers, buf[c][j] (c < k): its float2 field, its x and y planes, or
// its files, whose lengths go to len[c][j] and whose buffers hold `capacity` bytes each.
struct FlowDest {
    enum Kind { field, u8_planes, float_planes, jpeg_pair, png } kind;
    int k;
    void *const *buf[2];
    size_t *len[2];
    size_t capacity;
    int bound, quality;  // u8_planes and jpeg_pair: the quantisation bound; jpeg_pair: the JPEG quality
    // the float buffers also hold each pair's initial flow when use_initial_flow is set (the calc calls; the chains refuse it)
    bool warm;
    bool files() const { return kind == jpeg_pair || kind == png; }
    // an output array is null
    bool missing() const {
        for (int c = 0; c < k; ++c)
            if (!buf[c] || (files() && !len[c])) return true;
        return false;
    }
};
template <typename T> void *const *bytes_of(T *const *a) { return reinterpret_cast<void *const *>(a); }
FlowDest field_dest(float *const *f) { return {FlowDest::field, 1, {bytes_of(f), nullptr}, {}, 0, 0, 0, true}; }
FlowDest planes_dest(float *const *x, float *const *y, bool warm) {
    return {FlowDest::float_planes, 2, {bytes_of(x), bytes_of(y)}, {}, 0, 0, 0, warm};
}
FlowDest u8_dest(int bound, uint8_t *const *x, uint8_t *const *y) {
    return {FlowDest::u8_planes, 2, {bytes_of(x), bytes_of(y)}, {}, 0, bound, 0, false};
}
FlowDest png_dest(uint8_t *const *out, size_t capacity, size_t *len) {
    return {FlowDest::png, 1, {bytes_of(out), nullptr}, {len, nullptr}, capacity, 0, 0, false};
}
FlowDest jpeg_dest(int bound, int quality, uint8_t *const *x, uint8_t *const *y, size_t capacity, size_t *len_x, size_t *len_y) {
    return {FlowDest::jpeg_pair, 2, {bytes_of(x), bytes_of(y)}, {len_x, len_y}, capacity, bound, quality, false};
}

// the calls whose outputs hold no initial flow have none to read: refused before anything is enqueued
int refuse_initial_flow(dfb_handle *h, const FlowDest &d) {
    if (d.warm || !initial_flow(h)) return DFB_OK;
    return fail(h, DFB_ERR_INVALID_ARG,
                "use_initial_flow is set: only the calls that take a float flow buffer (dfb_calc_device / _host / _batch_host / _batch_device "
                "and their _planes forms) read an initial flow; set it to 0 for this call");
}

// Each of the M pairs' output buffers is present and host memory; `label` names them in the message.
int check_pair_outputs(dfb_handle *h, int M, const FlowDest &d, const char *label) {
    for (int j = 0; j < M; ++j)
        for (int c = 0; c < d.k; ++c)
            if (!d.buf[c][j] || host_pointer_kind(d.buf[c][j]) < 0)
                return null_flow(h, std::string(label) + " " + std::to_string(j) + " is null or a device pointer (host entry point)");
    return DFB_OK;
}

// Where the solve of pj writes its result: a float2 field with rows of `pitch` bytes, two float planes, or (bound > 0) two
// uint8 planes.  With init, the same float buffers hold the pair's initial flow: the solve reads it before it writes.
void bind_start(FlowAlgorithm::PairJob &pj, const float *x, const float *y, size_t pitch, int step) {
    pj.init_x = x;
    pj.init_y = y;
    pj.init_pitch = pitch / sizeof(float);
    pj.init_step = step;
}
void bind_field(FlowAlgorithm::PairJob &pj, float *f, size_t pitch, bool init) {
    pj.flow_xy = f;
    pj.flow_pitch_bytes = pitch;
    if (init) bind_start(pj, f, f + 1, pitch, 2);
}
void bind_planes(FlowAlgorithm::PairJob &pj, float *x, float *y, size_t pitch, bool init) {
    pj.fx = x;
    pj.fy = y;
    pj.f_pitch = pitch;
    if (init) bind_start(pj, x, y, pitch, 1);
}
void bind_u8(FlowAlgorithm::PairJob &pj, uint8_t *x, uint8_t *y, size_t pitch, int bound) {
    pj.bound = bound;
    pj.qx = x;
    pj.qy = y;
    pj.q_pitch = pitch;
}

// pinned staging buffers exist only for callers that pass pageable memory: allocated on first use
uint8_t *stage_frame(dfb_handle *h, int r) {
    h->h_frame[r].allocate((size_t)h->max_w * h->max_h);
    return h->h_frame[r];
}
// output pair p's staging buffer, px_bytes per pixel of the handle's maximum frame
uint8_t *stage_out(dfb_handle *h, int p, size_t px_bytes) {
    h->h_out[p].allocate((size_t)h->max_w * h->max_h * px_bytes);
    return h->h_out[p];
}

void ensure_streams(dfb_handle *h) {
    if (h->s_in) return;
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking));
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
    DFB_CUDA(cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking));
}

void ensure_fetch_stream(dfb_handle *h) {
    ensure_streams(h);
    if (!h->s_fetch) DFB_CUDA(cudaStreamCreateWithFlags(&h->s_fetch, cudaStreamNonBlocking));
}

// The x and y tables of a sw x sh -> dw x dh INTER_LINEAR resize (x: coefficients reset at the borders, y: rows clamped).
// A launch with the old tables may still be running on any stream when the geometry changes, hence the device sync.
const ResizeTap *ensure_taps(TapTable &t, int sw, int sh, int dw, int dh) {
    if (t.sw != sw || t.sh != sh || t.dw != dw || t.dh != dh) {
        std::vector<ResizeTap> xt, yt;
        build_resize_taps(dw, sw, true, xt);
        build_resize_taps(dh, sh, false, yt);
        DFB_CUDA(cudaDeviceSynchronize());
        t.d.allocate(sizeof(ResizeTap) * (dw + dh));
        DFB_CUDA(cudaMemcpy(t.d, xt.data(), sizeof(ResizeTap) * dw, cudaMemcpyHostToDevice));
        DFB_CUDA(cudaMemcpy(t.d + dw, yt.data(), sizeof(ResizeTap) * dh, cudaMemcpyHostToDevice));
        t.sw = sw;
        t.sh = sh;
        t.dw = dw;
        t.dh = dh;
    }
    return t.d;
}

// 1: device (or managed) memory a kernel may read and write
bool is_device_pointer(const void *p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Geometry of a call that resizes BGR frames: source sw x sh (packed BGR rows of bgr_pitch bytes), destination dw x dh, where
// 0 / 0 means no resize.  Resolves the destination and checks it against the handle's maximum.
int check_geometry(dfb_handle *h, int sw, int sh, size_t bgr_pitch, int &dw, int &dh) {
    if (sw <= 0 || sh <= 0 || dw < 0 || dh < 0 || (dw == 0) != (dh == 0) || bgr_pitch < (size_t)sw * 3)
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    if (dw == 0) {
        dw = sw;
        dh = sh;
    }
    return check_size(h, dw, dh);
}

// Y / Cb / Cr planes of one dw x dh frame in one scratch block, with room for whole 16 x 16 MCUs (YccExtent::mcu): 64-byte
// aligned rows, round16(dh) luma rows, and round8(ceil(dh / 2)) chroma rows of round8(ceil(dw / 2)) samples or more
struct YccLayout {
    size_t y_pitch, c_pitch, cb_off, cr_off, bytes;
    YccLayout(int dw, int dh) {
        const int cw = (dw + 1) / 2, crows = round_up((dh + 1) / 2, 8);
        y_pitch = (size_t)round_up(dw, 64);
        c_pitch = (size_t)round_up(cw, 64);
        cb_off = y_pitch * 2 * crows;
        cr_off = cb_off + c_pitch * crows;
        bytes = cr_off + c_pitch * crows;
    }
};

// the resize of a frame-extraction call: null tables mean no resize
const ResizeTap *ycc_tables(dfb_handle *h, int sw, int sh, int dw, int dh) {
    return (sw == dw && sh == dh) ? nullptr : ensure_taps(h->ycc_taps, sw, sh, dw, dh);
}

// the out(k, length) of a call that writes one file to out and its length to *out_len
auto single_out(uint8_t *out, size_t *out_len) {
    return [=](int, size_t n) {
        *out_len = n;
        return out;
    };
}

// the planes of a YccLayout block as a JPEG encoder reads them
JpegSrc ycc_src(const uint8_t *base, const YccLayout &L) {
    JpegSrc src;
    src.base = base;
    src.img_stride = L.bytes;
    src.pitch = L.y_pitch;
    src.cb_off = L.cb_off;
    src.cr_off = L.cr_off;
    src.c_pitch = L.c_pitch;
    return src;
}

// The JPEG files of a call, encoded in groups into two slots of up to `per_slot` files each, so one group can be read back
// while the next is encoded.  The handle's "jpeg_exact" picks the encoder: JpegExactEncoder, or nvJPEG with file k of slot s
// in encoder state s * per_slot + k.
class JpegSink {
  public:
    // slots: how many slots the call uses (1 or 2); always_exact: the call writes imencode's bytes whatever the handle says
    JpegSink(dfb_handle *h, int per_slot, int slots, bool always_exact = false) : h_(h), per_slot_(per_slot) {
        if (always_exact || h->jpeg_exact) {
            if (!h->jex) h->jex.reset(new JpegExactEncoder());
            jex_ = h->jex.get();
        } else {
            if (!h->jpeg) h->jpeg.reset(new JpegEncoder());
            h->jpeg->ensure_states(slots * per_slot);
        }
    }
    bool exact() const { return jex_ != nullptr; }
    // What the encoder reads of a w x h image: JpegExactEncoder replicates edge samples itself, except the padded chroma
    // columns; nvJPEG reads whole blocks (gray) or MCUs (colour), so the planes must hold libjpeg's padding up to there.
    YccExtent ycc_extent() const { return jex_ ? YccExtent::chroma_cols : YccExtent::mcu; }
    bool needs_padded_gray(int w, int hh) const { return !jex_ && (w % 8 || hh % 8); }
    // Enqueues the encodes of n images of src into `slot` on s, each file to be at most capacity bytes; the exact encoder's
    // lengths follow them to the host on s.
    void encode(int slot, int n, const JpegSrc &src, int components, int w, int hh, int quality, size_t capacity, cudaStream_t s) {
        group_[slot] = Group{src, components, w, hh, quality, capacity};
        if (jex_) {
            h_->alg->launches += jex_->encode(n, src, components, w, hh, quality, capacity, slot, s);
            return;
        }
        for (int k = 0; k < n; ++k) {
            const uint8_t *p = src.base + (size_t)k * src.img_stride;
            if (components == 1)
                h_->jpeg->enqueue(slot * per_slot_ + k, p, src.pitch, w, hh, quality, s);
            else
                h_->jpeg->enqueue_ycc420(slot * per_slot_ + k, p, src.pitch, p + src.cb_off, p + src.cr_off, src.c_pitch, w, hh, quality, s);
        }
    }
    // Once the slot's encode is complete: in file order, a file over capacity fails the call with
    // std::runtime_error(too_small(k, bytes it needs)) for the first such file k.  File k is copied to out(k, length) on s,
    // the bytes are added to d2h_bytes and s is synchronised.
    template <typename TooSmall, typename Out> void deliver(int slot, int n, TooSmall &&too_small, Out &&out, cudaStream_t s) {
        const Group &g = group_[slot];
        if (jex_) {
            auto reject = [&](int k, uint64_t reported) {
                return too_small(k, jex_->needed(reported, g.src, k, g.components, g.w, g.h, g.quality, s));
            };
            jex_->files().deliver(slot, n, g.capacity, reject, out, h_->counters.d2h_bytes, s);
            return;
        }
        for (int k = 0; k < n; ++k) {
            const int st = slot * per_slot_ + k;
            const size_t len = h_->jpeg->length(st, s);
            if (len > g.capacity) throw std::runtime_error(too_small(k, len));
            h_->jpeg->fetch(st, out(k, len), len, s);
            h_->counters.d2h_bytes += len;
        }
        DFB_CUDA(cudaStreamSynchronize(s));
    }

  private:
    struct Group {
        JpegSrc src;
        int components, w, h, quality;
        size_t capacity;
    };
    dfb_handle *h_;
    int per_slot_;
    JpegExactEncoder *jex_ = nullptr;
    Group group_[2] = {};
};

void ensure_png_scratch(dfb_handle *h) {
    if (h->png_scratch) return;
    h->png_scratch.allocate(png_pack_scratch_bytes());
    DFB_CUDA(cudaMemset(h->png_scratch, 0, png_pack_scratch_bytes()));
    DFB_CUDA(cudaDeviceSynchronize());
}

// Runs stage(g) for the groups g = 0..G-1 and finish(g - 1) after each, then finish(G - 1): the files of group g - 1 are read
// back while the GPU works on group g.
template <typename Stage, typename Finish> void run_groups(int G, Stage &&stage, Finish &&finish) {
    for (int g = 0; g < G; ++g) {
        stage(g);
        if (g > 0) finish(g - 1);
    }
    finish(G - 1);
}

// pair j of a batch: frames j and j + |step| (:315-316), in engine slots modulo nslots
FlowAlgorithm::PairJob pair_job(int j, int step, int nslots) {
    const int astep = std::abs(step);
    FlowAlgorithm::PairJob pj{};
    pj.slot_a = (step > 0 ? j : j + astep) % nslots;
    pj.slot_b = (step > 0 ? j + astep : j) % nslots;
    return pj;
}

// Enqueues on s the preparation of frames [prepared, last] of a dense array (frame f: w x hh bytes at frames + f * w * hh)
// into their engine slots, as one batch; prepared ends at last + 1.
void prepare_dense(FlowAlgorithm &alg, const uint8_t *frames, int w, int hh, int &prepared, int last, cudaStream_t s) {
    std::vector<const uint8_t *> srcs;
    std::vector<int> slots;
    for (; prepared <= last; ++prepared) {
        srcs.push_back(frames + (size_t)w * hh * prepared);
        slots.push_back(prepared % alg.num_slots());
    }
    if (!srcs.empty()) alg.prepare_frames((int)srcs.size(), srcs.data(), w, w, hh, slots.data(), s);
}

// cv::resize(INTER_LINEAR) of a device gray plane, enqueued on s; an equal size is a copy
void resize_gray(dfb_handle *h, const uint8_t *src, size_t src_pitch, int sw, int sh, uint8_t *dst, size_t dst_pitch, int dw, int dh,
                 cudaStream_t s) {
    if (sw == dw && sh == dh) {
        DFB_CUDA(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, sw, sh, cudaMemcpyDeviceToDevice, s));
        return;
    }
    const ResizeTap *taps = ensure_taps(h->gray_taps, sw, sh, dw, dh);
    launch_resize_u8(src, src_pitch, sw, sh, dst, dst_pitch, dw, dh, taps, taps + dw, s);
    ++h->alg->launches;
}

// Frame source of the calc calls: host frames through the handle's ring of kFrameRing device frames (pageable ones through
// pinned staging, one H2D per frame on s_in), then ONE batched preparation per sub-batch of at most kFrameRing frames on
// s_compute (the per-frame stages are launch-latency-bound; a ring slot is reused only after its frame has been prepared).
// Asked for the frames up to `last`, it uploads one more, so that frame's H2D overlaps the solve.
std::function<void(int)> upload_ring(dfb_handle *h, const uint8_t *const *frames, int n_frames, int w, int hh) {
    constexpr int FR = dfb_handle::kFrameRing;
    ensure_streams(h);
    h->d_frame_pitch = (size_t)round_up(h->max_w, 128);
    for (auto &f : h->d_frame) f.allocate(h->d_frame_pitch * h->max_h);
    h->ev_in.ensure(FR);
    h->ev_pyr.ensure(FR);
    return [=, uploaded = 0](int last) mutable {  // frames [0, uploaded) have H2D + preparation enqueued
        const size_t fbytes = (size_t)w * hh;
        const int nslots = h->alg->num_slots();
        last = std::min(last + 1, n_frames - 1);
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
            h->alg->prepare_frames(cnt, srcs, h->d_frame_pitch, w, hh, slots, h->s_compute);
            for (int i = 0; i < cnt; ++i) DFB_CUDA(cudaEventRecord(h->ev_pyr[(first + i) % FR], h->s_compute));
            uploaded += cnt;
        }
    };
}

// Frame source of the flow chains: produce(first, last) enqueues on s_in the work that leaves frames [first, last] in
// h->pb_frames (w x hh each, dense) and records h->chain_ev.frame[f] for each; frames are requested in order.  Asked for the
// frames up to `last`, it produces one more, so that frame's decode overlaps the solve.
std::function<void(int)> dense_frames(dfb_handle *h, int n_frames, int w, int hh, const std::function<void(int, int)> &produce) {
    h->pb_frames.grow((size_t)w * hh * n_frames);
    h->chain_ev.frame.ensure(n_frames);
    return [=, &produce, produced = 0, prepared = 0](int last) mutable {
        const int ahead = std::min(last + 1, n_frames - 1);
        if (produced <= ahead) {
            produce(produced, ahead);
            produced = ahead + 1;
        }
        DFB_CUDA(cudaStreamWaitEvent(h->s_compute, h->chain_ev.frame[last], 0));
        prepare_dense(*h->alg, h->pb_frames, w, hh, prepared, last, h->s_compute);
    };
}

// What the flow group loop does with the pairs it solves.  Group g fills output slot g & 1: its pair i is output pair
// p = slot * B + i, in h->flow_out.
struct FlowOutput {
    std::function<void(FlowAlgorithm::PairJob &, int p)> bind;  // where the solve writes output pair p
    std::function<void(int slot, int m)> pack;                  // optional: s_compute work on the solved group
    std::function<void(int j0, int m, int slot)> send;          // s_out: the group's outputs leave the slot
    std::function<void(int j0, int m, int slot)> finish;        // host, a group later: the results to the caller
    // optional (use_initial_flow): s_compute copy of pair j's initial flow into output pair p, which bind made the solve's start
    std::function<void(int j, int p)> load;
};

// FlowDest's field, float_planes and u8_planes: the k buffers of output pair p (px pixels of bpp bytes each) at
// (p k + c) px bpp in the slots.  Pair j's buffers go to buf[c][j] straight into page-locked memory when all of them are,
// else through the pair's pinned staging buffer, copied out once the slot has been read back.
FlowOutput host_output(dfb_handle *h, const FlowDest &d, int B, int w, int hh, size_t px) {
    const int k = d.k;
    const size_t bpp = d.kind == FlowDest::field ? 2 * sizeof(float) : d.kind == FlowDest::float_planes ? sizeof(float) : 1;
    const size_t bytes = (size_t)w * hh * bpp, row = (size_t)w * bpp;  // one buffer of a pair
    h->flow_out.grow(2 * B * k * px * bpp);
    auto slot_buf = [=](int p, int c) { return h->flow_out + ((size_t)p * k + c) * px * bpp; };
    auto direct = [=](int j) {
        for (int c = 0; c < k; ++c)
            if (!is_pinned_host(d.buf[c][j])) return false;
        return true;
    };
    const bool init = d.warm && initial_flow(h);
    FlowOutput o;
    o.bind = [=](FlowAlgorithm::PairJob &pj, int p) {
        float *x = reinterpret_cast<float *>(slot_buf(p, 0)), *y = reinterpret_cast<float *>(slot_buf(p, 1));
        if (d.kind == FlowDest::field) bind_field(pj, x, row, init);
        else if (d.kind == FlowDest::float_planes) bind_planes(pj, x, y, row, init);
        else bind_u8(pj, slot_buf(p, 0), slot_buf(p, 1), row, d.bound);
    };
    o.send = [=](int j0, int m, int slot) {
        for (int i = 0; i < m; ++i) {
            const int j = j0 + i, p = slot * B + i;
            const bool dir = direct(j);
            for (int c = 0; c < k; ++c) {
                void *dst = dir ? d.buf[c][j] : stage_out(h, p, k * bpp) + c * bytes;
                DFB_CUDA(cudaMemcpyAsync(dst, slot_buf(p, c), bytes, cudaMemcpyDeviceToHost, h->s_out));
            }
            h->counters.d2h_bytes += k * bytes;
        }
    };
    o.finish = [=](int j0, int m, int slot) {
        for (int i = 0; i < m; ++i)
            if (!direct(j0 + i)) {
                DFB_CUDA(cudaEventSynchronize(h->flow_ev.freed[slot]));
                for (int c = 0; c < k; ++c) std::memcpy(d.buf[c][j0 + i], h->h_out[slot * B + i] + c * bytes, bytes);
            }
    };
    // the pair's staging buffer is free: the read-back of the group that last used this slot has been copied out (finish)
    if (init)
        o.load = [=](int j, int p) {
            const bool dir = direct(j);
            for (int c = 0; c < k; ++c) {
                const void *src = d.buf[c][j];
                if (!dir) src = std::memcpy(stage_out(h, p, k * bpp) + c * bytes, src, bytes);
                DFB_CUDA(cudaMemcpyAsync(slot_buf(p, c), src, bytes, cudaMemcpyHostToDevice, h->s_compute));
            }
            h->counters.h2d_bytes += k * bytes;
        };
    return o;
}

// FlowDest's jpeg_pair (-st=jpg of a flow chain): pair j's two quantised planes as JPEGs, encoded on s_out as one batch per group
// (src/common.cpp:56-57) and read back on s_fetch
FlowOutput jpg_output(dfb_handle *h, const FlowDest &d, int B, int w, int hh) {
    // quantised planes: whole 8 x 8 blocks, so nvJPEG reads their edge padding (written by launch_pad_edges) and nothing else
    const int qw = round_up(w, 8), qh = round_up(hh, 8);
    const size_t qpx = (size_t)qw * qh;
    h->flow_out.grow(qpx * 2 * 2 * B);
    auto sink = std::make_shared<JpegSink>(h, 2 * B, 2);
    FlowOutput o;
    o.bind = [=](FlowAlgorithm::PairJob &pj, int p) {
        uint8_t *x = h->flow_out + (size_t)p * 2 * qpx;
        bind_u8(pj, x, x + qpx, (size_t)qw, d.bound);
    };
    o.send = [=](int, int m, int slot) {
        // the group's 2 m planes: plane 2 i + c of the slot is pair i's x (c = 0) or y
        JpegSrc src;
        src.base = h->flow_out + (size_t)slot * B * 2 * qpx;
        src.img_stride = qpx;
        src.pitch = (size_t)qw;
        if (sink->needs_padded_gray(w, hh)) {
            launch_pad_edges(const_cast<uint8_t *>(src.base), src.pitch, src.img_stride, 2 * m, w, hh, qw, qh, h->s_out);
            ++h->alg->launches;
        }
        sink->encode(slot, 2 * m, src, 1, w, hh, d.quality, d.capacity, h->s_out);
    };
    o.finish = [=](int j0, int m, int slot) {
        DFB_CUDA(cudaEventSynchronize(h->flow_ev.freed[slot]));
        auto too_small = [&](int, size_t need) {
            return "jpeg output buffer too small (" + std::to_string(need) + " > " + std::to_string(d.capacity) + ")";
        };
        auto out = [&](int k, size_t len) {
            const int j = j0 + (k >> 1);
            d.len[k & 1][j] = len;
            return static_cast<uint8_t *>(d.buf[k & 1][j]);
        };
        sink->deliver(slot, 2 * m, too_small, out, h->s_fetch);
    };
    return o;
}

// FlowDest's png (the -st=png branch of encode_save): the flow fields in the slot, convertFlowToPngImage (src/common.cpp:18-46)
// of each on s_compute, imencode(".png") (:66-71) of the group as one batch into encoder slot `slot` on s_out, read back on
// s_fetch.  px: pixels each pair's field reserves.
FlowOutput png_output(dfb_handle *h, const FlowDest &d, int B, int w, int hh, size_t px) {
    const size_t img = (size_t)3 * w * hh;
    h->flow_out.grow(2 * B * px * 2 * sizeof(float));
    h->png_bgr.grow(2 * B * img);
    ensure_png_scratch(h);
    if (!h->png) h->png.reset(new PngEncoder());
    auto field = [=](int p) { return reinterpret_cast<float *>(h->flow_out + (size_t)p * px * 2 * sizeof(float)); };
    FlowOutput o;
    o.bind = [=](FlowAlgorithm::PairJob &pj, int p) { bind_field(pj, field(p), (size_t)w * 2 * sizeof(float), false); };
    o.pack = [=](int slot, int m) {
        for (int p = slot * B; p < slot * B + m; ++p)
            launch_flow_to_png_image(field(p), (size_t)w * 8, w, hh, h->png_bgr + p * img, (size_t)w * 3, h->png_scratch, nullptr, h->s_compute);
        h->alg->launches += 2 * m;
    };
    o.send = [=](int, int m, int slot) {
        h->alg->launches += h->png->encode(m, h->png_bgr + slot * B * img, img, (size_t)w * 3, w, hh, slot, h->s_out);
    };
    o.finish = [=](int j0, int m, int slot) {
        DFB_CUDA(cudaEventSynchronize(h->flow_ev.freed[slot]));
        auto reject = [&](int i, uint64_t n) {
            if (n == 0) return "png encoder failed on pair " + std::to_string(j0 + i);
            return "png output buffer too small: pair " + std::to_string(j0 + i) + " needs " + std::to_string(n) + " bytes, capacity is " +
                   std::to_string(d.capacity);
        };
        auto to = [&](int i, size_t n) {
            d.len[0][j0 + i] = n;
            return static_cast<uint8_t *>(d.buf[0][j0 + i]);
        };
        h->png->files().deliver(slot, m, d.capacity, reject, to, h->counters.d2h_bytes, h->s_fetch);
    };
    return o;
}

// The output of d for groups of B pairs of w x hh, each pair's field or planes reserving px pixels of the slots
FlowOutput flow_output(dfb_handle *h, const FlowDest &d, int B, int w, int hh, size_t px) {
    if (d.kind == FlowDest::png) return png_output(h, d, B, w, hh, px);
    if (d.kind == FlowDest::jpeg_pair) return jpg_output(h, d, B, w, hh);
    return host_output(h, d, B, w, hh, px);
}

// The batch shape of calc_optflows_imp (src/denseflow_gpu.cpp:307-342): the M = n_frames - |step| pairs in groups of B on
// four streams, two groups in flight (the reference runs its stages as host threads around queues, include/dense_flow.h:76-80):
//   s_in      the frame source's copies and decodes; prepare(last) leaves frames up to `last` prepared in engine slots
//             f % num_slots(), ordered on s_compute
//   s_compute pyramids / polynomial expansions + flow of group g into output slot g & 1, then the output's pack
//   s_out     the output's read-back or encodes of the group
//   s_fetch   files of group g-1 to the host while the GPU works on group g
// Runs inside guarded(), for M > 0.
int flow_groups(dfb_handle *h, int n_frames, int step, int w, int hh, int B, const std::function<void(int)> &prepare,
                const FlowOutput &o) {
    const int astep = std::abs(step);
    const int M = n_frames - astep;  // :308
    ensure_fetch_stream(h);
    FlowAlgorithm &alg = *h->alg;
    alg.begin_batch();
    alg.ensure_slots(B + astep + 1);  // one group plus the look-ahead frame
    const int nslots = alg.num_slots();
    auto &ev = h->flow_ev;
    ev.solved.ensure(2);
    ev.freed.ensure(2);
    std::vector<FlowAlgorithm::PairJob> jobs(B);
    auto stage = [&](int g) {
        const int j0 = g * B, m = std::min(B, M - j0), slot = g & 1;
        prepare(j0 + m - 1 + astep);  // pairs j0..j0+m-1 touch frames j0..j0+m-1+|step| for either sign of step
        if (g >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev.freed[slot], 0));  // group g-2 has left the slot
        for (int i = 0; i < m; ++i) {
            jobs[i] = pair_job(j0 + i, step, nslots);
            o.bind(jobs[i], slot * B + i);
            if (o.load) o.load(j0 + i, slot * B + i);
        }
        alg.solve_batch(jobs.data(), m, w, hh, h->s_compute);
        if (o.pack) o.pack(slot, m);
        DFB_CUDA(cudaEventRecord(ev.solved[slot], h->s_compute));
        DFB_CUDA(cudaStreamWaitEvent(h->s_out, ev.solved[slot], 0));
        o.send(j0, m, slot);
        DFB_CUDA(cudaEventRecord(ev.freed[slot], h->s_out));
        h->counters.pairs += m;  // total_flows += 1 (:340)
    };
    auto finish = [&](int g) { o.finish(g * B, std::min(B, M - g * B), g & 1); };
    run_groups((M + B - 1) / B, stage, finish);
    DFB_CUDA(cudaStreamSynchronize(h->s_in));
    DFB_CUDA(cudaStreamSynchronize(h->s_compute));
    DFB_CUDA(cudaStreamSynchronize(h->s_out));
    return DFB_OK;
}

// The calc calls over host buffers: the pairs' outputs go where d says.  Runs inside guarded().
int batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int w, int hh, const FlowDest &d) {
    if (int rc = check_size(h, w, hh)) return rc;
    if (n_frames < 0 || !frames) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    const int M = std::max(n_frames - std::abs(step), 0);  // :308
    if (M == 0) return DFB_OK;
    for (int f = 0; f < n_frames; ++f)
        if (!frames[f] || host_pointer_kind(frames[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "frames[" + std::to_string(f) + "] is null or a device pointer (host entry point: use dfb_calc_batch_device)");
    if (int rc = check_pair_outputs(h, M, d, "output")) return rc;
    const int B = std::max(1, std::min(h->alg->max_concurrent_pairs(w, hh), dfb_handle::kMaxGroup));
    // output slots at the handle's maximum frame, so that calls of other sizes reuse them (a 1080p handle runs 7 pairs per
    // group, a 340x256 one up to 64)
    const size_t px = (size_t)h->max_w * h->max_h;
    return flow_groups(h, n_frames, step, w, hh, B, upload_ring(h, frames, n_frames, w, hh), flow_output(h, d, B, w, hh, px));
}

// dfb_calc_batch_host[_u8|_planes|_png]: the checks of the output arrays (`missing`: the message when one is null), then the call
int calc_batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int w, int hh, const FlowDest &d,
                    const char *missing) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (int rc = refuse_initial_flow(h, d)) return rc;
    if (d.kind == FlowDest::u8_planes && d.bound <= 0) return fail(h, DFB_ERR_INVALID_ARG, "bound should > 0!");  // check_param, src/denseflow_gpu.cpp:15-18
    if (n_frames > std::abs(step) && d.missing()) return null_flow(h, missing);
    return guarded(h, [&]() { return batch_host(h, frames, n_frames, step, w, hh, d); });
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
    if (!std::strcmp(name, "jpeg_exact")) {  // an output contract of the handle, not of the flow algorithm
        if (value != 0 && value != 1) return fail(h, DFB_ERR_INVALID_ARG, "jpeg_exact must be 0 or 1");
        h->jpeg_exact = value == 1;
        return DFB_OK;
    }
    if (!h->alg->set_param(name, value)) return fail(h, DFB_ERR_INVALID_ARG, std::string("bad parameter ") + name);
    return DFB_OK;
}

int dfb_get_param(const dfb_handle *h, const char *name, double *value) {
    if (!h || !name || !value) return DFB_ERR_INVALID_ARG;
    if (!std::strcmp(name, "jpeg_exact")) {
        *value = h->jpeg_exact ? 1 : 0;
        return DFB_OK;
    }
    return h->alg->get_param(name, value) ? DFB_OK : DFB_ERR_INVALID_ARG;
}

int dfb_calc_device(dfb_handle *h, const uint8_t *a, size_t a_pitch, const uint8_t *b, size_t b_pitch, int width,
                    int height, float *flow_xy, size_t flow_pitch, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!flow_xy) return null_flow(h, "null buffer");
    if (!a || !b) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (int rc = check_size(h, width, height)) return rc;
    if (a_pitch < (size_t)width || b_pitch < (size_t)width || flow_pitch < (size_t)width * 8)
        return fail(h, DFB_ERR_INVALID_ARG, "pitch smaller than a row");
    if ((reinterpret_cast<uintptr_t>(flow_xy) | flow_pitch) & 7)
        return fail(h, DFB_ERR_INVALID_ARG, "flow_xy and flow_pitch must be 8-byte aligned (CV_32FC2 rows)");
    return guarded(h, [&]() {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        h->alg->begin_batch();
        const int slots[2] = {0, 1};  // one call per frame: the two frames' rows may lie at different pitches
        h->alg->prepare_frames(1, &a, a_pitch, width, height, slots, s);
        h->alg->prepare_frames(1, &b, b_pitch, width, height, slots + 1, s);
        FlowAlgorithm::PairJob pj{0, 1};
        bind_field(pj, flow_xy, flow_pitch, initial_flow(h));  // the start is read on s before the solve writes the field
        h->alg->solve_batch(&pj, 1, width, height, s);
        ++h->counters.pairs;
        return DFB_OK;
    });
}

int dfb_calc_host(dfb_handle *h, const uint8_t *a, const uint8_t *b, int width, int height, float *flow_xy) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!flow_xy) return null_flow(h, "null buffer");
    if (!a || !b) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    const uint8_t *frames[2] = {a, b};
    float *flows[1] = {flow_xy};
    return guarded(h, [&]() { return batch_host(h, frames, 2, 1, width, height, field_dest(flows)); });
}

int dfb_calc_batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                        float *const *flows) {
    return calc_batch_host(h, frames, n_frames, step, width, height, field_dest(flows), "flows is null");
}

int dfb_calc_batch_host_u8(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                           int bound, uint8_t *const *qx, uint8_t *const *qy) {
    return calc_batch_host(h, frames, n_frames, step, width, height, u8_dest(bound, qx, qy), "qx/qy is null");
}

int dfb_calc_batch_host_planes(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                               float *const *fx, float *const *fy) {
    return calc_batch_host(h, frames, n_frames, step, width, height, planes_dest(fx, fy, true), "fx/fy is null");
}

int dfb_calc_batch_host_png(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height, uint8_t *const *png,
                            size_t capacity, size_t *len) {
    return calc_batch_host(h, frames, n_frames, step, width, height, png_dest(png, capacity, len), "png / len is null");
}

}  // extern "C"

namespace {

// dfb_calc_batch_device[_planes]: pair j's flow to out + j * 2 w h floats, as one float2 field or (planar) as the x plane
// followed by the y plane
int batch_device(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height, float *flows, bool planar,
                 void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (int rc = check_size(h, width, height)) return rc;
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    const int astep = std::abs(step);
    const int M = std::max(n_frames - astep, 0);
    if (M == 0) return DFB_OK;
    if (!flows) return null_flow(h, "null buffer");
    if (!frames) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    const bool init = initial_flow(h);
    return guarded(h, [&]() {
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
            prepare_dense(alg, frames, width, height, prepared, j0 + m - 1 + astep, s);
            for (int i = 0; i < m; ++i) {
                const int j = j0 + i;
                jobs[i] = pair_job(j, step, nslots);
                float *out = flows + (size_t)j * fbytes * 2;  // with init it holds the pair's initial flow
                if (planar) bind_planes(jobs[i], out, out + fbytes, (size_t)width * sizeof(float), init);
                else bind_field(jobs[i], out, (size_t)width * 2 * sizeof(float), init);
            }
            alg.solve_batch(jobs.data(), m, width, height, s);
            h->counters.pairs += m;
        }
        return DFB_OK;
    });
}

}  // namespace

extern "C" {

int dfb_calc_batch_device(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                          float *flows, void *stream) {
    return batch_device(h, frames, n_frames, step, width, height, flows, false, stream);
}

int dfb_calc_batch_device_planes(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                                 float *planes, void *stream) {
    return batch_device(h, frames, n_frames, step, width, height, planes, true, stream);
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
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        ensure_png_scratch(h);
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
        resize_gray(h, src, src_pitch, sw, sh, dst, dst_pitch, dw, dh, static_cast<cudaStream_t>(stream));
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
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        JpegSink sink(h, 1, 1);
        JpegSrc src;
        src.base = gray;
        src.pitch = gray_pitch;
        if (!sink.exact()) {
            // nvJPEG gets a copy in handle scratch: it refuses some pitches of block-aligned planes (status 2), and it must not
            // read the caller's bytes around the plane.  Partial blocks are padded as libjpeg pads them.
            const int pw = round_up(width, 8), ph = round_up(height, 8);
            const size_t pitch = (size_t)round_up(pw, 64);
            h->enc_gray.grow(pitch * ph);
            DFB_CUDA(cudaMemcpy2DAsync(h->enc_gray, pitch, gray, gray_pitch, width, height, cudaMemcpyDeviceToDevice, s));
            if (sink.needs_padded_gray(width, height)) {
                launch_pad_edges(h->enc_gray, pitch, 0, 1, width, height, pw, ph, s);
                ++h->alg->launches;
            }
            src.base = h->enc_gray;
            src.pitch = pitch;
        }
        sink.encode(0, 1, src, 1, width, height, quality, out_capacity, s);
        DFB_CUDA(cudaStreamSynchronize(s));
        auto too_small = [&](int, size_t need) {
            return std::string(sink.exact() ? "jpeg output" : "nvjpeg: output") + " buffer too small (" + std::to_string(need) + " > " +
                   std::to_string(out_capacity) + ")";
        };
        sink.deliver(0, 1, too_small, single_out(out, out_len), s);
        return DFB_OK;
    });
}

int dfb_encode_jpeg_gray_batch_device(dfb_handle *h, const uint8_t *planes, size_t pitch, size_t plane_stride, int n, int width,
                                      int height, int quality, uint8_t *const *out, size_t capacity, size_t *len, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (n < 0) return fail(h, DFB_ERR_INVALID_ARG, "n must be >= 0");
    if (n == 0) return DFB_OK;
    if (!planes || !out || !len) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (width <= 0 || height <= 0 || width > 65535 || height > 65535 || pitch < (size_t)width || quality < 1 || quality > 100 ||
        (n > 1 && plane_stride < pitch * (size_t)(height - 1) + (size_t)width))
        return fail(h, DFB_ERR_INVALID_ARG, "bad geometry or quality");
    if (capacity == 0) return fail(h, DFB_ERR_INVALID_ARG, "zero capacity");
    if (!is_device_pointer(planes)) return fail(h, DFB_ERR_INVALID_ARG, "planes must be device memory (device entry point)");
    for (int i = 0; i < n; ++i)
        if (!out[i] || host_pointer_kind(out[i]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "jpeg output " + std::to_string(i) + " is null or a device pointer (host entry point)");
    return guarded(h, [&]() {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        JpegSink sink(h, n, 1, true);
        JpegSrc src;
        src.base = planes;
        src.pitch = pitch;
        src.img_stride = plane_stride;
        sink.encode(0, n, src, 1, width, height, quality, capacity, s);
        DFB_CUDA(cudaStreamSynchronize(s));
        auto too_small = [&](int i, size_t need) {
            return "jpeg output buffer too small: plane " + std::to_string(i) + " (" + std::to_string(need) + " > " + std::to_string(capacity) + ")";
        };
        auto to = [&](int i, size_t n) {
            len[i] = n;
            return out[i];
        };
        sink.deliver(0, n, too_small, to, s);
        return DFB_OK;
    });
}

int dfb_decode_jpeg_gray_device(dfb_handle *h, const uint8_t *jpeg, size_t jpeg_len, uint8_t *gray, size_t gray_pitch, int max_width,
                                int max_height, int *width, int *height, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!jpeg || !jpeg_len || !gray || !width || !height) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    return guarded(h, [&]() {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (!h->jpeg) h->jpeg.reset(new JpegEncoder());
        int w = 0, hh = 0, nc = 0;
        h->jpeg->image_info(jpeg, jpeg_len, &w, &hh, &nc);
        *width = w;
        *height = hh;
        if (w <= 0 || hh <= 0) return fail(h, DFB_ERR_INVALID_ARG, "not a JPEG image");
        if (w > max_width || hh > max_height || gray_pitch < (size_t)w)
            return fail(h, DFB_ERR_SIZE, "decoded frame " + std::to_string(w) + "x" + std::to_string(hh) + " does not fit the output buffer");
        h->dec_bgr.grow((size_t)w * hh * 3);
        // imread(IMREAD_COLOR) -> BGR, then the decode stage's cvtColor(BGR2GRAY) (src/denseflow_gpu.cpp:160-163), bit-exact from there on
        h->jpeg->decode_bgr(jpeg, jpeg_len, h->dec_bgr, (size_t)w * 3, w, hh, s);
        launch_bgr_to_gray(h->dec_bgr, (size_t)w * 3, w, hh, gray, gray_pitch, s);
        ++h->alg->launches;
        return (int)DFB_OK;
    });
}

}  // extern "C"

namespace {

// The per-batch chain after decode: gray frames (sw x sh, resized to dw x dh) by `produce` (dense_frames) -> flow -> the
// output of `d`: quantise and two JPEGs per pair, convertFlowToPngImage and one PNG per pair, or the two float planes of each
// pair.  Runs inside guarded().
int process_chain(dfb_handle *h, int n_frames, int step, int dw, int dh, const FlowDest &d, const std::function<void(int, int)> &produce) {
    const int B = std::max(1, std::min(h->alg->max_concurrent_pairs(dw, dh), 8));
    return flow_groups(h, n_frames, step, dw, dh, B, dense_frames(h, n_frames, dw, dh, produce), flow_output(h, d, B, dw, dh, (size_t)dw * dh));
}

// Every file of a JPEG batch parsed on the host; an unsupported or corrupt header is the call's error.
int parse_jpegs(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n, std::vector<JpegHeader> &hd) {
    hd.resize(n);
    for (int i = 0; i < n; ++i) {
        if (!jpeg[i] || !len[i]) return fail(h, DFB_ERR_INVALID_ARG, "frame " + std::to_string(i) + ": null or empty JPEG buffer");
        if (host_pointer_kind(jpeg[i]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "frame " + std::to_string(i) + ": the JPEG bytes must be in host memory");
        try {
            hd[i] = parse_jpeg_header(jpeg[i], len[i], i);
        } catch (const JpegUnsupported &e) {
            return fail(h, DFB_ERR_UNSUPPORTED, e.what());
        } catch (const std::exception &e) {
            return fail(h, DFB_ERR_INVALID_ARG, e.what());
        }
    }
    return DFB_OK;
}

// The files of a JPEG batch parsed, and all of one size: *sw / *sh receive it (n > 0).
int parse_jpegs_one_size(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n, std::vector<JpegHeader> &hd, int &sw, int &sh) {
    if (int rc = parse_jpegs(h, jpeg, len, n, hd)) return rc;
    sw = hd[0].w;
    sh = hd[0].h;
    for (int f = 1; f < n; ++f)
        if (hd[f].w != sw || hd[f].h != sh)
            return fail(h, DFB_ERR_SIZE, "frame " + std::to_string(f) + " is " + std::to_string(hd[f].w) + "x" + std::to_string(hd[f].h) +
                                             ", frame 0 is " + std::to_string(sw) + "x" + std::to_string(sh) + " (one size per batch)");
    return DFB_OK;
}

// The checks both flow chains make first, in this order: use_initial_flow, the frame array, step, bound, the requested size
// (0 / 0: none).
int check_chain_args(dfb_handle *h, bool frames_null, int n_frames, int step, const FlowDest &d, int dw, int dh) {
    if (int rc = refuse_initial_flow(h, d)) return rc;
    if (frames_null || n_frames < 0) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    if (step == 0) return fail(h, DFB_ERR_INVALID_ARG, "step must be non-zero for flow extraction");
    if (d.kind == FlowDest::jpeg_pair && d.bound <= 0) return fail(h, DFB_ERR_INVALID_ARG, "bound should > 0!");
    if (dw < 0 || dh < 0 || (dw == 0) != (dh == 0)) return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    return DFB_OK;
}

// dfb_process_bgr_batch_host[_png|_planes]: the checks, then the chain with decoded BGR frames as its source; `label` names the
// pairs' outputs in the messages
int bgr_chain(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int sw, int sh, int dw, int dh, const FlowDest &d,
              const char *label) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (int rc = check_chain_args(h, !bgr, n_frames, step, d, dw, dh)) return rc;
    if (int rc = check_geometry(h, sw, sh, (size_t)sw * 3, dw, dh)) return rc;
    const int M = std::max(n_frames - std::abs(step), 0);
    if (M == 0) return DFB_OK;
    if (d.missing()) return fail(h, DFB_ERR_INVALID_ARG, "null output");
    for (int f = 0; f < n_frames; ++f)
        if (!bgr[f] || host_pointer_kind(bgr[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "bgr[" + std::to_string(f) + "] is null or a device pointer (host entry point)");
    if (int rc = check_pair_outputs(h, M, d, label)) return rc;
    return guarded(h, [&]() {
        // frame source: H2D of BGR frame f into staging buffer f & 1 -> cvtColor -> resize (decode stage tail, :163-170)
        const size_t fpx = (size_t)dw * dh, bgr_bytes = (size_t)sw * sh * 3;
        h->pb_bgr.grow(2 * bgr_bytes);  // two staging frames: H2D of f+1 overlaps gray/resize of f
        h->pb_gray.grow((size_t)sw * sh);
        h->chain_ev.gray.ensure(2);
        auto produce = [&](int first, int last) {
            auto &ev = h->chain_ev;
            for (int f = first; f <= last; ++f) {
                const int sb = f & 1;
                if (f >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_in, ev.gray[sb], 0));
                uint8_t *stage = h->pb_bgr + (size_t)sb * bgr_bytes;
                DFB_CUDA(cudaMemcpyAsync(stage, bgr[f], bgr_bytes, cudaMemcpyHostToDevice, h->s_in));
                h->counters.h2d_bytes += bgr_bytes;
                uint8_t *dst = h->pb_frames + fpx * f;
                if (dw == sw && dh == sh) {
                    launch_bgr_to_gray(stage, (size_t)sw * 3, sw, sh, dst, dw, h->s_in);
                } else {
                    launch_bgr_to_gray(stage, (size_t)sw * 3, sw, sh, h->pb_gray, sw, h->s_in);
                    resize_gray(h, h->pb_gray, sw, sw, sh, dst, dw, dw, dh, h->s_in);
                }
                h->alg->launches += 1;
                DFB_CUDA(cudaEventRecord(ev.gray[sb], h->s_in));
                DFB_CUDA(cudaEventRecord(ev.frame[f], h->s_in));
            }
        };
        return process_chain(h, n_frames, step, dw, dh, d, produce);
    });
}

// dfb_process_jpeg_batch_host[_png|_planes]: the checks, then the chain with JPEG files decoded on the device as its source
int jpeg_chain(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n_frames, int step, int dw, int dh, const FlowDest &d,
               const char *label) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (int rc = check_chain_args(h, !jpeg || !len, n_frames, step, d, dw, dh)) return rc;
    const int M = std::max(n_frames - std::abs(step), 0);
    if (M == 0) return DFB_OK;
    std::vector<JpegHeader> hd;
    int sw = 0, sh = 0;
    if (int rc = parse_jpegs_one_size(h, jpeg, len, n_frames, hd, sw, sh)) return rc;
    if (int rc = check_geometry(h, sw, sh, (size_t)sw * 3, dw, dh)) return rc;
    if (d.missing()) return fail(h, DFB_ERR_INVALID_ARG, "null output");
    if (int rc = check_pair_outputs(h, M, d, label)) return rc;
    return guarded(h, [&]() {
        if (!h->jdec) h->jdec.reset(new JpegDecoder());
        // frame source: the requested frames are decoded as one group, straight into the gray frame array when no resize is
        // asked for, else into scratch and resized frame by frame; only the compressed bytes cross PCIe
        const size_t fpx = (size_t)dw * dh, spx = (size_t)sw * sh;
        auto produce = [&](int first, int last) {
            const int m = last - first + 1;
            const bool resize = dw != sw || dh != sh;
            if (resize) {
                DFB_CUDA(cudaStreamSynchronize(h->s_in));  // the previous group's resizes have read the scratch
                h->pb_gray.grow(spx * m);
            }
            uint8_t *dst = resize ? h->pb_gray : h->pb_frames + fpx * first;
            h->jdec->decode(jpeg + first, len + first, hd.data() + first, m, 1, dst, sw, spx, h->s_in, first);
            h->alg->launches += h->jdec->launches;
            for (int f = first; f <= last; ++f) {
                h->counters.h2d_bytes += len[f];
                if (resize) resize_gray(h, h->pb_gray + spx * (f - first), sw, sw, sh, h->pb_frames + fpx * f, dw, dw, dh, h->s_in);
                DFB_CUDA(cudaEventRecord(h->chain_ev.frame[f], h->s_in));
            }
        };
        return process_chain(h, n_frames, step, dw, dh, d, produce);
    });
}

constexpr int kExtractGroup = 8;  // frames per group of the -s=0 pipeline

// The frame source of the -s=0 pipeline: source(g, f0, m, convert) enqueues the work that leaves the BGR of group g's frames
// f0 .. f0 + m - 1 readable by s_compute, and calls convert(i, bgr) for frame f0 + i once it is.
using ConvertFrame = std::function<void(int, const uint8_t *)>;
using FrameSource = std::function<void(int, int, int, const ConvertFrame &)>;

// extract_frames_video's batch (src/denseflow_gpu.cpp:82-144: resize + imencode(".jpg") per frame) of n_frames sw x sh BGR frames
// on four streams, groups of G frames in flight:
//   s_in      the frame source: the group's frames to BGR in h->ex_bgr (room for `staging` frames)
//   s_compute resize + YCbCr 4:2:0 of each frame into the planes of its group
//   s_out     the group's encodes, as one batch
//   s_fetch   files of group g-1 to the host while the GPU works on group g
// Runs inside guarded().
int extract_frames(dfb_handle *h, int n_frames, int sw, int sh, int dw, int dh, int quality, uint8_t *const *jpg, size_t capacity,
                   size_t *len, int staging, const FrameSource &source) {
    constexpr int G = kExtractGroup;
    ensure_fetch_stream(h);
    const YccLayout L(dw, dh);
    h->ex_bgr.grow((size_t)staging * sw * sh * 3);
    h->ex_ycc.grow(2 * G * L.bytes);
    const ResizeTap *taps = ycc_tables(h, sw, sh, dw, dh);
    auto &ev = h->extract_ev;
    for (Events *e : {&ev.h2d, &ev.conv, &ev.planes, &ev.enc}) e->ensure(2);
    JpegSink sink(h, G, 2);

    auto convert_group = [&](int g) {
        const int f0 = g * G, m = std::min(G, n_frames - f0), slot = g & 1;
        uint8_t *planes = h->ex_ycc + (size_t)slot * G * L.bytes;
        if (g >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev.enc[slot], 0));  // group g-2's planes have been encoded
        source(g, f0, m, [&](int i, const uint8_t *bgr) {
            uint8_t *p = planes + (size_t)i * L.bytes;
            launch_bgr_to_ycc420(bgr, (size_t)sw * 3, sw, sh, dw, dh, taps, taps ? taps + dw : nullptr, p, L.y_pitch, p + L.cb_off,
                                 p + L.cr_off, L.c_pitch, h->s_compute, sink.ycc_extent());
            ++h->alg->launches;
        });
        DFB_CUDA(cudaEventRecord(ev.planes[slot], h->s_compute));
        DFB_CUDA(cudaStreamWaitEvent(h->s_out, ev.planes[slot], 0));
        sink.encode(slot, m, ycc_src(planes, L), 3, dw, dh, quality, capacity, h->s_out);
        DFB_CUDA(cudaEventRecord(ev.enc[slot], h->s_out));
    };
    auto finish_group = [&](int g) {
        const int f0 = g * G, m = std::min(G, n_frames - f0);
        DFB_CUDA(cudaEventSynchronize(ev.enc[g & 1]));
        auto too_small = [&](int i, size_t need) {
            return "jpeg output buffer too small: frame " + std::to_string(f0 + i) + " needs " + std::to_string(need) + " bytes, capacity is " +
                   std::to_string(capacity);
        };
        auto out = [&](int i, size_t n) {
            len[f0 + i] = n;
            return jpg[f0 + i];
        };
        sink.deliver(g & 1, m, too_small, out, h->s_fetch);
    };
    run_groups((n_frames + G - 1) / G, convert_group, finish_group);
    DFB_CUDA(cudaStreamSynchronize(h->s_in));
    DFB_CUDA(cudaStreamSynchronize(h->s_compute));
    DFB_CUDA(cudaStreamSynchronize(h->s_out));
    return DFB_OK;
}

}  // namespace

extern "C" {

int dfb_process_bgr_batch_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int sw, int sh, int dw, int dh,
                               int bound, int jpeg_quality, uint8_t *const *jpg_x, uint8_t *const *jpg_y, size_t capacity,
                               size_t *len_x, size_t *len_y) {
    return bgr_chain(h, bgr, n_frames, step, sw, sh, dw, dh, jpeg_dest(bound, jpeg_quality, jpg_x, jpg_y, capacity, len_x, len_y),
                     "jpeg output");
}

int dfb_process_bgr_batch_host_png(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int sw, int sh, int dw, int dh,
                                   uint8_t *const *png, size_t capacity, size_t *len) {
    return bgr_chain(h, bgr, n_frames, step, sw, sh, dw, dh, png_dest(png, capacity, len), "png output");
}

int dfb_process_jpeg_batch_host(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n_frames, int step, int dw, int dh,
                                int bound, int jpeg_quality, uint8_t *const *jpg_x, uint8_t *const *jpg_y, size_t capacity,
                                size_t *len_x, size_t *len_y) {
    return jpeg_chain(h, jpeg, len, n_frames, step, dw, dh, jpeg_dest(bound, jpeg_quality, jpg_x, jpg_y, capacity, len_x, len_y),
                      "jpeg output");
}

int dfb_process_jpeg_batch_host_png(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int step, int dw,
                                    int dh, uint8_t *const *png, size_t capacity, size_t *len) {
    return jpeg_chain(h, jpeg, jpeg_len, n_frames, step, dw, dh, png_dest(png, capacity, len), "png output");
}

int dfb_process_bgr_batch_host_planes(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int sw, int sh, int dw, int dh,
                                      float *const *fx, float *const *fy) {
    return bgr_chain(h, bgr, n_frames, step, sw, sh, dw, dh, planes_dest(fx, fy, false), "plane output");
}

int dfb_process_jpeg_batch_host_planes(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int step, int dw,
                                       int dh, float *const *fx, float *const *fy) {
    return jpeg_chain(h, jpeg, jpeg_len, n_frames, step, dw, dh, planes_dest(fx, fy, false), "plane output");
}

int dfb_new_size(int width, int height, int new_width, int new_height, int new_short, int *dw, int *dh) {
    if (!dw || !dh) return fail(nullptr, DFB_ERR_INVALID_ARG, "null output");
    // check_param (src/denseflow_gpu.cpp:27-35)
    if (new_height < 0 || new_width < 0 || new_short < 0) return fail(nullptr, DFB_ERR_INVALID_ARG, "height and width cannot < 0!");
    if (new_short > 0 && new_height + new_width != 0) return fail(nullptr, DFB_ERR_INVALID_ARG, "do not set height and width when set short!");
    if (width <= 0 || height <= 0) return fail(nullptr, DFB_ERR_INVALID_ARG, "width/height must be positive");
    // get_new_size (:62-79): (int)round(...) of the scaled side
    auto scaled = [](int a, int b, int n) { return (int)std::round(a * 1.0 / b * n); };
    *dw = width;
    *dh = height;
    if (new_width > 0 && new_height > 0) {
        *dw = new_width;
        *dh = new_height;
    } else if (new_width > 0) {
        *dw = new_width;
        *dh = scaled(height, width, new_width);
    } else if (new_height > 0) {
        *dw = scaled(width, height, new_height);
        *dh = new_height;
    } else if (new_short > 0 && std::min(width, height) > new_short) {
        if (width < height) {
            *dw = new_short;
            *dh = scaled(height, width, new_short);
        } else {
            *dw = scaled(width, height, new_short);
            *dh = new_short;
        }
    }
    return DFB_OK;
}

int dfb_jpeg_info(const uint8_t *jpeg, size_t len, int *width, int *height) {
    if (!jpeg || !len || !width || !height) return fail(nullptr, DFB_ERR_INVALID_ARG, "null or empty JPEG buffer");
    try {
        const JpegHeader hd = parse_jpeg_header(jpeg, len, 0);
        *width = hd.w;
        *height = hd.h;
        return DFB_OK;
    } catch (const JpegUnsupported &e) {
        return fail(nullptr, DFB_ERR_UNSUPPORTED, e.what());
    } catch (const std::exception &e) {
        return fail(nullptr, DFB_ERR_INVALID_ARG, e.what());
    }
}

int dfb_decode_jpeg_batch_device(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n, int channels, uint8_t *out,
                                 size_t pitch, size_t frame_stride, int max_width, int max_height, int *width, int *height, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (n < 0) return fail(h, DFB_ERR_INVALID_ARG, "n must be >= 0");
    if (n == 0) return DFB_OK;
    if (!jpeg || !len || !out) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (channels != 1 && channels != 3) return fail(h, DFB_ERR_INVALID_ARG, "channels must be 1 (gray) or 3 (BGR)");
    if (!is_device_pointer(out)) return fail(h, DFB_ERR_INVALID_ARG, "out must be device memory (device entry point)");
    std::vector<JpegHeader> hd;
    if (int rc = parse_jpegs(h, jpeg, len, n, hd)) return rc;
    for (int i = 0; i < n; ++i) {
        if (width) width[i] = hd[i].w;
        if (height) height[i] = hd[i].h;
    }
    for (int i = 0; i < n; ++i)
        if (hd[i].w > max_width || hd[i].h > max_height || pitch < (size_t)hd[i].w * channels ||
            (n > 1 && frame_stride < pitch * hd[i].h))
            return fail(h, DFB_ERR_SIZE, "frame " + std::to_string(i) + ": " + std::to_string(hd[i].w) + "x" + std::to_string(hd[i].h) +
                                             " does not fit the output (" + std::to_string(max_width) + "x" + std::to_string(max_height) +
                                             ", pitch " + std::to_string(pitch) + ", frame stride " + std::to_string(frame_stride) + ")");
    return guarded(h, [&]() {
        if (!h->jdec) h->jdec.reset(new JpegDecoder());
        h->jdec->decode(jpeg, len, hd.data(), n, channels, out, pitch, frame_stride, static_cast<cudaStream_t>(stream));
        h->alg->launches += h->jdec->launches;
        for (int i = 0; i < n; ++i) h->counters.h2d_bytes += len[i] - hd[i].data_off;
        return DFB_OK;
    });
}

int dfb_debug_jpeg_coefficients(dfb_handle *h, const uint8_t *jpeg, size_t len, int16_t *out, size_t capacity_blocks, int *n_blocks,
                                int *sync_rounds) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!jpeg || !out || !n_blocks) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    std::vector<JpegHeader> hd;
    if (int rc = parse_jpegs(h, &jpeg, &len, 1, hd)) return rc;
    *n_blocks = hd[0].blocks();
    if ((size_t)hd[0].blocks() > capacity_blocks)
        return fail(h, DFB_ERR_SIZE, "the file has " + std::to_string(hd[0].blocks()) + " blocks, capacity is " + std::to_string(capacity_blocks));
    return guarded(h, [&]() {
        if (!h->jdec) h->jdec.reset(new JpegDecoder());
        h->jdec->coefficients(jpeg, len, hd[0], out, nullptr);
        if (sync_rounds) *sync_rounds = h->jdec->sync_rounds;
        return DFB_OK;
    });
}

int dfb_bgr_to_ycc420_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int src_width, int src_height, int dst_width,
                             int dst_height, uint8_t *y, size_t y_pitch, uint8_t *cb, uint8_t *cr, size_t c_pitch, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || !y || !cb || !cr) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    int dw = dst_width, dh = dst_height;
    if (int rc = check_geometry(h, src_width, src_height, bgr_pitch, dw, dh)) return rc;
    if (y_pitch < (size_t)dw || c_pitch < (size_t)(dw + 1) / 2) return fail(h, DFB_ERR_INVALID_ARG, "pitch smaller than a row");
    for (const void *p : {(const void *)bgr, (const void *)y, (const void *)cb, (const void *)cr})
        if (!is_device_pointer(p)) return fail(h, DFB_ERR_INVALID_ARG, "bgr / y / cb / cr must be device memory (device entry point)");
    return guarded(h, [&]() {
        const ResizeTap *taps = ycc_tables(h, src_width, src_height, dw, dh);
        launch_bgr_to_ycc420(bgr, bgr_pitch, src_width, src_height, dw, dh, taps, taps ? taps + dw : nullptr, y, y_pitch, cb, cr, c_pitch,
                             static_cast<cudaStream_t>(stream));
        ++h->alg->launches;
        return DFB_OK;
    });
}

size_t dfb_jpeg_max_bytes_bgr(int width, int height) {
    if (width <= 0 || height <= 0) return 0;
    // 2 bytes per sample of the MCU-padded image: 16 x 16 luma MCUs carry 256 Y and 2 x 64 chroma samples
    const size_t wp = (size_t)round_up(width, 16), hp = (size_t)round_up(height, 16);
    return (wp * hp * 3 / 2) * 2 + 4096;
}

int dfb_encode_jpeg_bgr_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int src_width, int src_height, int dst_width,
                               int dst_height, int quality, uint8_t *out, size_t out_capacity, size_t *out_len, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || !out || !out_len) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    int dw = dst_width, dh = dst_height;
    if (int rc = check_geometry(h, src_width, src_height, bgr_pitch, dw, dh)) return rc;
    if (quality < 1 || quality > 100) return fail(h, DFB_ERR_INVALID_ARG, "quality must be in 1..100");
    if (!is_device_pointer(bgr)) return fail(h, DFB_ERR_INVALID_ARG, "bgr must be device memory (device entry point)");
    if (host_pointer_kind(out) < 0) return fail(h, DFB_ERR_INVALID_ARG, "out must be host memory");
    return guarded(h, [&]() {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        const YccLayout L(dw, dh);
        h->enc_ycc.grow(L.bytes);
        const ResizeTap *taps = ycc_tables(h, src_width, src_height, dw, dh);
        JpegSink sink(h, 1, 1);
        uint8_t *p = h->enc_ycc;
        launch_bgr_to_ycc420(bgr, bgr_pitch, src_width, src_height, dw, dh, taps, taps ? taps + dw : nullptr, p, L.y_pitch, p + L.cb_off,
                             p + L.cr_off, L.c_pitch, s, sink.ycc_extent());
        ++h->alg->launches;
        sink.encode(0, 1, ycc_src(p, L), 3, dw, dh, quality, out_capacity, s);
        DFB_CUDA(cudaStreamSynchronize(s));
        auto too_small = [&](int, size_t need) {
            return "jpeg output buffer too small: the bitstream needs " + std::to_string(need) + " bytes, capacity is " + std::to_string(out_capacity);
        };
        sink.deliver(0, 1, too_small, single_out(out, out_len), s);
        return DFB_OK;
    });
}

int dfb_extract_frames_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int src_width, int src_height, int dst_width,
                            int dst_height, int quality, uint8_t *const *jpg, size_t capacity, size_t *len) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || n_frames < 0) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    int dw = dst_width, dh = dst_height;
    if (int rc = check_geometry(h, src_width, src_height, (size_t)src_width * 3, dw, dh)) return rc;
    if (quality < 1 || quality > 100) return fail(h, DFB_ERR_INVALID_ARG, "quality must be in 1..100");
    if (n_frames == 0) return DFB_OK;
    if (!jpg || !len) return fail(h, DFB_ERR_INVALID_ARG, "null output");
    for (int f = 0; f < n_frames; ++f) {
        if (!bgr[f] || host_pointer_kind(bgr[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "bgr[" + std::to_string(f) + "] is null or a device pointer (host entry point)");
        if (!jpg[f] || host_pointer_kind(jpg[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "jpeg output " + std::to_string(f) + " is null or a device pointer (host entry point)");
    }
    const int sw = src_width, sh = src_height;
    return guarded(h, [&]() {
        // frame source: H2D of frame f into staging frame f & 1, interleaved with the converts
        const size_t bgr_bytes = (size_t)sw * sh * 3;
        auto upload = [&](int, int f0, int m, const ConvertFrame &convert) {
            auto &ev = h->extract_ev;
            for (int i = 0; i < m; ++i) {
                const int f = f0 + i, sb = f & 1;
                uint8_t *stage = h->ex_bgr + sb * bgr_bytes;
                if (f >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_in, ev.conv[sb], 0));
                DFB_CUDA(cudaMemcpyAsync(stage, bgr[f], bgr_bytes, cudaMemcpyHostToDevice, h->s_in));
                DFB_CUDA(cudaEventRecord(ev.h2d[sb], h->s_in));
                h->counters.h2d_bytes += bgr_bytes;
                DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev.h2d[sb], 0));
                convert(i, stage);
                DFB_CUDA(cudaEventRecord(ev.conv[sb], h->s_compute));
            }
        };
        return extract_frames(h, n_frames, sw, sh, dw, dh, quality, jpg, capacity, len, 2, upload);
    });
}

int dfb_extract_frames_jpeg_host(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int dst_width,
                                 int dst_height, int quality, uint8_t *const *jpg, size_t capacity, size_t *len) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!jpeg || !jpeg_len || n_frames < 0) return fail(h, DFB_ERR_INVALID_ARG, "frames is null");
    int dw = dst_width, dh = dst_height;
    if (dw < 0 || dh < 0 || (dw == 0) != (dh == 0)) return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    if (quality < 1 || quality > 100) return fail(h, DFB_ERR_INVALID_ARG, "quality must be in 1..100");
    if (n_frames == 0) return DFB_OK;
    if (!jpg || !len) return fail(h, DFB_ERR_INVALID_ARG, "null output");
    for (int f = 0; f < n_frames; ++f)
        if (!jpg[f] || host_pointer_kind(jpg[f]) < 0)
            return fail(h, DFB_ERR_INVALID_ARG, "jpeg output " + std::to_string(f) + " is null or a device pointer (host entry point)");
    std::vector<JpegHeader> hd;
    int sw = 0, sh = 0;
    if (int rc = parse_jpegs_one_size(h, jpeg, jpeg_len, n_frames, hd, sw, sh)) return rc;
    if (int rc = check_geometry(h, sw, sh, (size_t)sw * 3, dw, dh)) return rc;
    return guarded(h, [&]() {
        if (!h->jdec) h->jdec.reset(new JpegDecoder());
        // frame source: imdecode of group g to BGR into staging slot g & 1 (the host waits for the decoder's status)
        constexpr int G = kExtractGroup;
        const size_t bgr_bytes = (size_t)sw * sh * 3;
        auto decode = [&](int g, int f0, int m, const ConvertFrame &convert) {
            auto &ev = h->extract_ev;
            const int slot = g & 1;
            uint8_t *stage = h->ex_bgr + (size_t)slot * G * bgr_bytes;
            if (g >= 2) DFB_CUDA(cudaStreamWaitEvent(h->s_in, ev.planes[slot], 0));  // group g-2's frames have been converted
            h->jdec->decode(jpeg + f0, jpeg_len + f0, hd.data() + f0, m, 3, stage, (size_t)sw * 3, bgr_bytes, h->s_in, f0);
            h->alg->launches += h->jdec->launches;
            for (int i = 0; i < m; ++i) h->counters.h2d_bytes += jpeg_len[f0 + i];
            DFB_CUDA(cudaEventRecord(ev.h2d[slot], h->s_in));
            DFB_CUDA(cudaStreamWaitEvent(h->s_compute, ev.h2d[slot], 0));
            for (int i = 0; i < m; ++i) convert(i, stage + (size_t)i * bgr_bytes);
        };
        return extract_frames(h, n_frames, sw, sh, dw, dh, quality, jpg, capacity, len, 2 * G, decode);
    });
}

size_t dfb_png_max_bytes(int width, int height) { return png_max_bytes(width, height); }

int dfb_encode_png_bgr_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int width, int height, uint8_t *out, size_t out_capacity,
                              size_t *out_len, void *stream) {
    if (!h) return DFB_ERR_INVALID_ARG;
    if (!bgr || !out || !out_len) return fail(h, DFB_ERR_INVALID_ARG, "null buffer");
    if (width <= 0 || height <= 0 || bgr_pitch < (size_t)width * 3) return fail(h, DFB_ERR_INVALID_ARG, "bad geometry");
    if (int rc = check_size(h, width, height)) return rc;
    if (!is_device_pointer(bgr)) return fail(h, DFB_ERR_INVALID_ARG, "bgr must be device memory (device entry point)");
    if (host_pointer_kind(out) < 0) return fail(h, DFB_ERR_INVALID_ARG, "out must be host memory");
    return guarded(h, [&]() {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (!h->png) h->png.reset(new PngEncoder());
        h->alg->launches += h->png->encode(1, bgr, 0, bgr_pitch, width, height, 0, s);
        DFB_CUDA(cudaStreamSynchronize(s));
        auto reject = [&](int, uint64_t len) {
            if (len == 0) return std::string("png encoder failed");
            return "png output buffer too small: the file needs " + std::to_string(len) + " bytes, capacity is " + std::to_string(out_capacity);
        };
        h->png->files().deliver(0, 1, out_capacity, reject, single_out(out, out_len), h->counters.d2h_bytes, s);
        return DFB_OK;
    });
}

int dfb_debug_run_kernel(dfb_handle *h, const char *kernel, const float *const *in, int n_in, float *const *out, int n_out, int width,
                         int height, const double *scalars, int n_scalars, double *scalars_out) {
    if (!h || !kernel) return DFB_ERR_INVALID_ARG;
    if (width <= 0 || height <= 0 || n_in < 0 || n_out < 0 || n_in > 16 || n_out > 16) return fail(h, DFB_ERR_INVALID_ARG, "bad arguments");
    return guarded(h, [&]() {
        const std::string k(kernel);
        if (h->alg->debug_run(k, in, n_in, out, n_out, width, height, scalars, n_scalars, scalars_out)) return DFB_OK;  // the engine's own stages
        auto sc = [&](int i) { return i < n_scalars ? scalars[i] : 0.0; };
        if (k == "jpeg_padded_gray" || k == "jpeg_padded_ycc420") {  // the planes the nvJPEG path hands the encoder
            const bool gray = k == "jpeg_padded_gray";
            if (n_in != (gray ? 1 : 3) || n_out != n_in) throw std::runtime_error(k + ": expects " + std::to_string(gray ? 1 : 3) + " inputs and outputs");
            const size_t px = (size_t)width * height;
            std::vector<uint8_t> host(px * n_in);
            for (size_t i = 0; i < px; ++i)  // gray, or packed BGR from the B, G, R planes
                for (int c = 0; c < n_in; ++c) host[i * n_in + c] = (uint8_t)std::lrint(std::min(std::max(in[c][i], 0.f), 255.f));
            auto download = [&](float *dst, const uint8_t *src, size_t pitch, int w, int hh) {
                std::vector<uint8_t> b((size_t)w * hh);
                DFB_CUDA(cudaMemcpy2D(b.data(), w, src, pitch, w, hh, cudaMemcpyDeviceToHost));
                for (size_t i = 0; i < b.size(); ++i) dst[i] = b[i];
            };
            DeviceBuffer<uint8_t> src, planes;
            src.allocate(host.size());
            DFB_CUDA(cudaMemcpy(src, host.data(), host.size(), cudaMemcpyHostToDevice));
            if (gray) {
                const int pw = round_up(width, 8), ph = round_up(height, 8);
                planes.allocate((size_t)pw * ph);
                DFB_CUDA(cudaMemcpy2D(planes, pw, src, width, width, height, cudaMemcpyDeviceToDevice));
                launch_pad_edges(planes, pw, 0, 1, width, height, pw, ph, nullptr);
                download(out[0], planes, pw, pw, ph);
                return DFB_OK;
            }
            const int dw = sc(0) > 0 ? (int)sc(0) : width, dh = sc(1) > 0 ? (int)sc(1) : height;
            const YccLayout L(dw, dh);
            planes.allocate(L.bytes);
            const ResizeTap *taps = ycc_tables(h, width, height, dw, dh);
            uint8_t *p = planes;
            launch_bgr_to_ycc420(src, (size_t)width * 3, width, height, dw, dh, taps, taps ? taps + dw : nullptr, p, L.y_pitch, p + L.cb_off,
                                 p + L.cr_off, L.c_pitch, nullptr, YccExtent::mcu);
            const int cw = round_up((dw + 1) / 2, 8), ch = round_up((dh + 1) / 2, 8);
            download(out[0], p, L.y_pitch, 2 * cw, 2 * ch);
            download(out[1], p + L.cb_off, L.c_pitch, cw, ch);
            download(out[2], p + L.cr_off, L.c_pitch, cw, ch);
            return DFB_OK;
        }
        if (k == "png_encode_batch") {  // n images through one PngEncoder::encode call, as the -st=png batch path runs them
            const int n = (int)sc(0);
            if (n_in != 3 || n_out != 1) throw std::runtime_error(k + ": expects 3 inputs and 1 output");
            if (n < 1 || n > 16 || height % n) throw std::runtime_error(k + ": n must be 1..16 and divide the height");
            const int hh = height / n;
            const size_t px = (size_t)width * height, cap = png_max_bytes(width, hh);
            std::vector<uint8_t> host(px * 3);
            for (size_t i = 0; i < px; ++i)  // packed BGR from the B, G, R planes
                for (int c = 0; c < 3; ++c) host[i * 3 + c] = (uint8_t)std::lrint(std::min(std::max(in[c][i], 0.f), 255.f));
            DeviceBuffer<uint8_t> src;
            src.allocate(host.size());
            DFB_CUDA(cudaMemcpy(src, host.data(), host.size(), cudaMemcpyHostToDevice));
            if (!h->png) h->png.reset(new PngEncoder());
            h->alg->launches += h->png->encode(n, src, (size_t)3 * width * hh, (size_t)3 * width, width, hh, 0, nullptr);
            DFB_CUDA(cudaStreamSynchronize(nullptr));
            std::vector<uint8_t> files((size_t)n * cap);
            auto reject = [&](int i, uint64_t len) { return "png encoder failed on image " + std::to_string(i) + " (" + std::to_string(len) + " bytes)"; };
            auto to = [&](int i, size_t len) {
                if (scalars_out) scalars_out[i] = (double)len;
                return files.data() + (size_t)i * cap;
            };
            h->png->files().deliver(0, n, cap, reject, to, h->counters.d2h_bytes, nullptr);
            for (size_t i = 0; i < files.size(); ++i) out[0][i] = files[i];  // out[0]: n rows of png_max_bytes(w, h / n)
            return DFB_OK;
        }
        int ow = width, oh = height;
        if (k == "resize") {
            ow = (int)sc(0);
            oh = (int)sc(1);
            if (ow <= 0 || oh <= 0) throw std::runtime_error("resize: bad destination size");
        }
        const int pitch = round_up(width, 32), opitch = round_up(ow, 32);
        std::deque<DeviceBuffer<float>> dev;
        auto alloc = [&](int w_, int h_, int p_) {
            DeviceBuffer<float> &b = dev.emplace_back();
            b.allocate((size_t)p_ * (h_ + 1) * sizeof(float));
            const Plane p{b, w_, h_, p_};
            fill_plane(p, 0);
            return p;
        };
        std::vector<Plane> pin, pout;
        for (int i = 0; i < n_in; ++i) {
            pin.push_back(alloc(width, height, pitch));
            upload_rows(pin[i], in[i], 0);
        }
        DeviceBuffer<double> d_part, d_sum;  // estimate_u's energy partials and their sum, when asked for
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
                d_part.allocate(sizeof(double) * nblk);
                d_sum.allocate(sizeof(double));
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
        } else if (k == "estimate_u_gamma") {  // estimate_u's inputs with p31, p32 after p22 and u3 after u2; scalars + gamma
            need(13, 3);
            const Tvl1Consts c{(float)sc(0), 0.f, (float)sc(1)};
            const bool calc = sc(2) != 0;
            const int nblk = estimate_u_blocks(width, height);
            if (calc) {
                d_part.allocate(sizeof(double) * nblk);
                d_sum.allocate(sizeof(double));
            }
            launch_estimate_u_gamma(pin[0], pin[1], pin[2], pin[3], &pin[4], pin[10], pin[11], pin[12], c, (float)sc(3), d_part, nullptr);
            if (calc) {
                launch_sum_partials(d_part, nblk, d_sum, nullptr);
                if (scalars_out) DFB_CUDA(cudaMemcpy(scalars_out, d_sum, sizeof(double), cudaMemcpyDeviceToHost));
            }
            inplace_from = 10;
        } else if (k == "estimate_dual_gamma") {  // u1, u2, u3, p11 .. p32
            need(9, 6);
            const Tvl1Consts c{0.f, (float)sc(0), 0.f};
            launch_estimate_dual_gamma(pin[0], pin[1], pin[2], &pin[3], c, nullptr);
            inplace_from = 3;
        } else if (k == "resize") {
            need(1, 1);
            pout = {alloc(ow, oh, opitch)};
            launch_resize_linear(pin[0], pout[0], (float)sc(2), (float)sc(3), n_scalars > 4 ? (float)sc(4) : 1.0f, nullptr);
        } else {
            throw std::runtime_error("unknown debug kernel " + k);
        }
        DFB_CUDA(cudaDeviceSynchronize());
        for (int i = 0; i < n_out; ++i) download_rows(out[i], inplace_from >= 0 ? pin[inplace_from + i] : pout[i], 0);
        return DFB_OK;
    });
}

int dfb_debug_time_kernel(dfb_handle *h, const char *kernel, int width, int height, int sets, int reps, double *ms_per_launch) {
    if (!h || !kernel || !ms_per_launch) return DFB_ERR_INVALID_ARG;
    if (width <= 0 || height <= 0 || sets < 1 || sets > 64 || reps < 1) return fail(h, DFB_ERR_INVALID_ARG, "bad arguments");
    return guarded(h, [&]() {
        const std::string k(kernel);
        const bool primal = k == "estimate_u";
        if (!primal && k != "estimate_dual") throw std::runtime_error("unknown kernel " + k);
        const int nplanes = primal ? 10 : 6;
        const int pitch = round_up(width, 32);
        const size_t pe = (size_t)pitch * (height + 1);
        DeviceBuffer<float> buf;
        buf.allocate(pe * sizeof(float) * nplanes * sets);
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
        Events ev(cudaEventDefault);
        ev.ensure(2);
        DFB_CUDA(cudaEventRecord(ev[0], nullptr));
        for (int i = 0; i < reps; ++i) run((i + 3) % sets);
        DFB_CUDA(cudaEventRecord(ev[1], nullptr));
        DFB_CUDA(cudaEventSynchronize(ev[1]));
        float ms = 0.f;
        DFB_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        *ms_per_launch = (double)ms / reps;
        return DFB_OK;
    });
}

int dfb_get_tvl1_stats(dfb_handle *h, dfb_tvl1_stats *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        h->alg->tvl1_stats(out);
        return DFB_OK;
    });
}

int dfb_get_tvl1_pair_stats(dfb_handle *h, int pair_index, dfb_tvl1_stats *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
        if (!h->alg->pair_stats(pair_index, out)) return fail(h, DFB_ERR_INVALID_ARG, "pair_index is not one of the last 256 pairs of the most recent tvl1 batch call");
        return (int)DFB_OK;
    });
}

int dfb_get_counters(dfb_handle *h, dfb_counters *out) {
    if (!h || !out) return DFB_ERR_INVALID_ARG;
    return guarded(h, [&]() {
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
