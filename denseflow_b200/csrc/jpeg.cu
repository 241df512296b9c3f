// jpeg.cu — GPU JPEG encode of the quantised flow planes through nvJPEG (SURVEY §8 f2): replaces the two
// imencode(".jpg", flow_img_x / flow_img_y, ...) calls of encodeFlowMap (/root/reference/src/common.cpp:56-57) with
// OpenCV's defaults (quality 95, baseline sequential, one gray component).  Byte identity with libjpeg-turbo is
// not a goal here (lossy) — the decoded planes are compared in the tests; jpeg_encode.cu is the byte-exact encoder behind
// the handle parameter "jpeg_exact".
// nvJPEG is loaded lazily with dlopen so the engine itself never depends on it.
#include <dlfcn.h>
#include <nvjpeg.h>

#include <mutex>
#include <vector>

#include "jpeg.h"

namespace dfb {

namespace {

struct Api {
    void *lib = nullptr;
    decltype(&nvjpegCreateSimple) CreateSimple = nullptr;
    decltype(&nvjpegDestroy) Destroy = nullptr;
    decltype(&nvjpegEncoderStateCreate) StateCreate = nullptr;
    decltype(&nvjpegEncoderStateDestroy) StateDestroy = nullptr;
    decltype(&nvjpegEncoderParamsCreate) ParamsCreate = nullptr;
    decltype(&nvjpegEncoderParamsDestroy) ParamsDestroy = nullptr;
    decltype(&nvjpegEncoderParamsSetQuality) SetQuality = nullptr;
    decltype(&nvjpegEncoderParamsSetSamplingFactors) SetSampling = nullptr;
    decltype(&nvjpegEncoderParamsSetOptimizedHuffman) SetOptHuff = nullptr;
    decltype(&nvjpegEncodeYUV) EncodeYUV = nullptr;
    decltype(&nvjpegEncodeRetrieveBitstream) Retrieve = nullptr;
    decltype(&nvjpegJpegStateCreate) JpegStateCreate = nullptr;
    decltype(&nvjpegJpegStateDestroy) JpegStateDestroy = nullptr;
    decltype(&nvjpegGetImageInfo) GetImageInfo = nullptr;
    decltype(&nvjpegDecode) Decode = nullptr;
};

Api &api() {
    static Api a;
    static std::once_flag once;
    std::call_once(once, [] {
        for (const char *name : {"libnvjpeg.so.12", "libnvjpeg.so", "/usr/local/cuda/lib64/libnvjpeg.so.12"}) {
            a.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
            if (a.lib) break;
        }
        if (!a.lib) return;
#define DFB_SYM(field, sym) a.field = reinterpret_cast<decltype(a.field)>(dlsym(a.lib, #sym))
        DFB_SYM(CreateSimple, nvjpegCreateSimple);
        DFB_SYM(Destroy, nvjpegDestroy);
        DFB_SYM(StateCreate, nvjpegEncoderStateCreate);
        DFB_SYM(StateDestroy, nvjpegEncoderStateDestroy);
        DFB_SYM(ParamsCreate, nvjpegEncoderParamsCreate);
        DFB_SYM(ParamsDestroy, nvjpegEncoderParamsDestroy);
        DFB_SYM(SetQuality, nvjpegEncoderParamsSetQuality);
        DFB_SYM(SetSampling, nvjpegEncoderParamsSetSamplingFactors);
        DFB_SYM(SetOptHuff, nvjpegEncoderParamsSetOptimizedHuffman);
        DFB_SYM(EncodeYUV, nvjpegEncodeYUV);
        DFB_SYM(Retrieve, nvjpegEncodeRetrieveBitstream);
        DFB_SYM(JpegStateCreate, nvjpegJpegStateCreate);
        DFB_SYM(JpegStateDestroy, nvjpegJpegStateDestroy);
        DFB_SYM(GetImageInfo, nvjpegGetImageInfo);
        DFB_SYM(Decode, nvjpegDecode);
#undef DFB_SYM
    });
    return a;
}

void check(nvjpegStatus_t st, const char *what) {
    if (st != NVJPEG_STATUS_SUCCESS) throw std::runtime_error(std::string("nvjpeg: ") + what + " failed with status " + std::to_string((int)st));
}

}  // namespace

struct JpegEncoder::Impl {
    nvjpegHandle_t handle = nullptr;
    std::vector<nvjpegEncoderState_t> states;
    nvjpegEncoderParams_t params = nullptr;
    int quality = -1;
    // colour frames: parameters of their own, so the gray path's sampling factors are never touched (created on first use)
    nvjpegEncoderParams_t params420 = nullptr;
    int quality420 = -1;
    nvjpegJpegState_t dec_state = nullptr;  // created on the first decode
};

JpegEncoder::JpegEncoder() : impl_(new Impl) {
    Api &a = api();
    if (!a.lib || !a.CreateSimple || !a.EncodeYUV || !a.Retrieve) throw std::runtime_error("nvjpeg: libnvjpeg.so.12 could not be loaded");
    check(a.CreateSimple(&impl_->handle), "nvjpegCreateSimple");
    check(a.ParamsCreate(impl_->handle, &impl_->params, nullptr), "nvjpegEncoderParamsCreate");
    ensure_states(1);
}

JpegEncoder::~JpegEncoder() {
    Api &a = api();
    if (impl_->params) a.ParamsDestroy(impl_->params);
    if (impl_->params420) a.ParamsDestroy(impl_->params420);
    for (auto st : impl_->states)
        if (st) a.StateDestroy(st);
    if (impl_->dec_state && a.JpegStateDestroy) a.JpegStateDestroy(impl_->dec_state);
    if (impl_->handle) a.Destroy(impl_->handle);
    delete impl_;
}

void JpegEncoder::ensure_states(int n) {
    Api &a = api();
    while ((int)impl_->states.size() < n) {
        nvjpegEncoderState_t st = nullptr;
        check(a.StateCreate(impl_->handle, &st, nullptr), "nvjpegEncoderStateCreate");
        impl_->states.push_back(st);
    }
}

void JpegEncoder::enqueue(int state, const uint8_t *gray, size_t pitch, int w, int h, int quality, cudaStream_t s) {
    Api &a = api();
    ensure_states(state + 1);
    if (quality != impl_->quality) {
        check(a.SetQuality(impl_->params, quality, s), "SetQuality");
        check(a.SetSampling(impl_->params, NVJPEG_CSS_GRAY, s), "SetSamplingFactors");
        check(a.SetOptHuff(impl_->params, 0, s), "SetOptimizedHuffman");
        impl_->quality = quality;
    }
    nvjpegImage_t img{};
    img.channel[0] = const_cast<unsigned char *>(gray);
    img.pitch[0] = pitch;
    check(a.EncodeYUV(impl_->handle, impl_->states[state], impl_->params, &img, NVJPEG_CSS_GRAY, w, h, s), "nvjpegEncodeYUV");
}

void JpegEncoder::enqueue_ycc420(int state, const uint8_t *y, size_t y_pitch, const uint8_t *cb, const uint8_t *cr, size_t c_pitch, int w,
                                 int h, int quality, cudaStream_t s) {
    Api &a = api();
    ensure_states(state + 1);
    if (!impl_->params420) check(a.ParamsCreate(impl_->handle, &impl_->params420, nullptr), "nvjpegEncoderParamsCreate");
    if (quality != impl_->quality420) {
        check(a.SetQuality(impl_->params420, quality, s), "SetQuality");
        check(a.SetSampling(impl_->params420, NVJPEG_CSS_420, s), "SetSamplingFactors");
        check(a.SetOptHuff(impl_->params420, 0, s), "SetOptimizedHuffman");
        impl_->quality420 = quality;
    }
    nvjpegImage_t img{};
    img.channel[0] = const_cast<unsigned char *>(y);
    img.pitch[0] = y_pitch;
    img.channel[1] = const_cast<unsigned char *>(cb);
    img.pitch[1] = c_pitch;
    img.channel[2] = const_cast<unsigned char *>(cr);
    img.pitch[2] = c_pitch;
    check(a.EncodeYUV(impl_->handle, impl_->states[state], impl_->params420, &img, NVJPEG_CSS_420, w, h, s), "nvjpegEncodeYUV");
}

size_t JpegEncoder::length(int state, cudaStream_t s) {
    size_t len = 0;
    check(api().Retrieve(impl_->handle, impl_->states.at(state), nullptr, &len, s), "RetrieveBitstream(size)");
    return len;
}

void JpegEncoder::fetch(int state, uint8_t *out, size_t len, cudaStream_t s) {
    check(api().Retrieve(impl_->handle, impl_->states.at(state), out, &len, s), "RetrieveBitstream");
}

void JpegEncoder::image_info(const uint8_t *jpeg, size_t len, int *w, int *h, int *components) {
    Api &a = api();
    if (!a.GetImageInfo) throw std::runtime_error("nvjpeg: decode entry points are missing");
    int nc = 0, ws[NVJPEG_MAX_COMPONENT] = {}, hs[NVJPEG_MAX_COMPONENT] = {};
    nvjpegChromaSubsampling_t css;
    check(a.GetImageInfo(impl_->handle, jpeg, len, &nc, &css, ws, hs), "nvjpegGetImageInfo");
    *w = ws[0];
    *h = hs[0];
    if (components) *components = nc;
}

void JpegEncoder::decode_bgr(const uint8_t *jpeg, size_t len, uint8_t *bgr, size_t pitch, int w, int h, cudaStream_t s) {
    Api &a = api();
    if (!a.Decode || !a.JpegStateCreate) throw std::runtime_error("nvjpeg: decode entry points are missing");
    if (!impl_->dec_state) check(a.JpegStateCreate(impl_->handle, &impl_->dec_state), "nvjpegJpegStateCreate");
    (void)w;
    (void)h;
    nvjpegImage_t out{};
    out.channel[0] = bgr;
    out.pitch[0] = pitch;
    check(a.Decode(impl_->handle, impl_->dec_state, jpeg, len, NVJPEG_OUTPUT_BGRI, &out, s), "nvjpegDecode");
}

}  // namespace dfb
