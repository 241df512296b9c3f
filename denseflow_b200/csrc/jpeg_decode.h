// jpeg_decode.h — batched JPEG decode on the GPU, exactly the pixels of cv2.imdecode(buf, IMREAD_COLOR) (libjpeg-turbo's
// default decompression: islow IDCT, fancy upsampling, YCbCr -> BGR) for baseline / extended sequential Huffman files.
#pragma once

#include <stdexcept>
#include <string>
#include <vector>

#include "common.cuh"

namespace dfb {

// A file outside the accepted subset (progressive, arithmetic, 12-bit, multi-scan, RGB / CMYK, 4:1:1, EXIF rotation): the
// message names the feature.  Corrupt data is reported as std::runtime_error naming the frame.
struct JpegUnsupported : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// Marker-level description of one file (host parse; see jpeg_decode.cu).
struct JpegHeader {
    int w = 0, h = 0, ncomp = 0, hmax = 1, vmax = 1, mcux = 0, mcuy = 0, bpm = 0, ri = 0, nseg = 0;
    int comp_h[3] = {}, comp_v[3] = {}, comp_q[3] = {}, comp_dc[3] = {}, comp_ac[3] = {};
    int32_t quant[4][64] = {};  // natural order, as the IDCT multiplies them (16-bit)
    bool has_quant[4] = {};
    struct Table {
        bool defined = false;
        uint8_t counts[16] = {};
        uint8_t symbols[256] = {};
    } dc[4], ac[4];
    size_t data_off = 0;  // first byte of the entropy-coded data
    int blocks() const { return mcux * mcuy * bpm; }
};

// Throws JpegUnsupported / std::runtime_error (prefixed with "frame <index>: ").
JpegHeader parse_jpeg_header(const uint8_t *buf, size_t len, int index);

class JpegDecoder {
  public:
    JpegDecoder() = default;
    ~JpegDecoder();
    JpegDecoder(const JpegDecoder &) = delete;
    JpegDecoder &operator=(const JpegDecoder &) = delete;

    // Decodes n parsed files.  channels 3: packed BGR rows; 1: cvtColor(BGR2GRAY) of them.  Frame i goes to
    // out + i * frame_stride with rows `pitch` bytes apart.  Enqueued on s; blocks until the device has reported every frame's
    // status and throws std::runtime_error naming the first corrupt frame as index_base + i.
    void decode(const uint8_t *const *jpeg, const size_t *len, const JpegHeader *hd, int n, int channels, uint8_t *out, size_t pitch,
                size_t frame_stride, cudaStream_t s, int index_base = 0);
    // Test hook: runs only the entropy decode and the DC prefix sums of one file; coefficients in decode (MCU) order, natural
    // order, absolute DC, are copied to the host buffer out (hd.blocks() x 64 int16).
    void coefficients(const uint8_t *jpeg, size_t len, const JpegHeader &hd, int16_t *out, cudaStream_t s);

    int sync_rounds = 0;  // re-decode rounds of the last call until the subsequence states stopped changing
    int launches = 0;     // kernels launched by the last call

  private:
    void run_entropy(const uint8_t *const *jpeg, const size_t *len, const JpegHeader *hd, int n, cudaStream_t s);
    void check_status(int n, cudaStream_t s, int index_base = 0);

    // grown on demand
    DeviceBuffer<uint8_t> d_ws;    // device workspace
    PinnedBuffer<uint8_t> h_stage;  // staging of the descriptors and file bytes
    PinnedBuffer<int> h_flag;      // the change flag of the sync rounds, then the frame status words
    // layout of the current call inside d_ws
    struct Layout;
    Layout *L = nullptr;
};

}  // namespace dfb
