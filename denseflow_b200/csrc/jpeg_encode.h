// jpeg_encode.h — imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q]) on the GPU, byte-identical to libjpeg-turbo with
// OpenCV's defaults (baseline, standard Huffman tables, islow DCT, no restart markers), for one gray component or
// YCbCr 4:2:0.  See jpeg_encode.cu.
#pragma once

#include <memory>

#include "file_slots.h"

namespace dfb {

// Device planes of a batch: image i's planes start at base + i * img_stride.  Gray: one plane at +0 (pitch bytes per row).
// YCbCr 4:2:0: Y at +0 (pitch), Cb / Cr at +cb_off / +cr_off (c_pitch), each chroma row holding jpeg_chroma_cols(w)
// samples (launch_bgr_to_ycc420 with that chroma width writes them).
struct JpegSrc {
    const uint8_t *base = nullptr;
    size_t img_stride = 0, pitch = 0;
    size_t cb_off = 0, cr_off = 0, c_pitch = 0;
};

// chroma columns the 4:2:0 encode reads: ceil(w / 2) rounded up to whole blocks; the columns past ceil(w / 2) are
// downsampled from the replicated last full-resolution column, as libjpeg's compressor pads its input
inline int jpeg_chroma_cols(int w) { return ((w + 1) / 2 + 7) / 8 * 8; }

// Bit 63 of a length: the file did not fit and the value is a lower bound (entropy data before byte stuffing).
constexpr uint64_t kJpegLenLowerBound = uint64_t(1) << 63;

// Workspace and output files, grown on demand.  Never touches nvJPEG.
class JpegExactEncoder {
  public:
    JpegExactEncoder() = default;
    JpegExactEncoder(const JpegExactEncoder &) = delete;
    JpegExactEncoder &operator=(const JpegExactEncoder &) = delete;
    // Encodes n w x h images (components 1 or 3) enqueued on s.  File i goes to files().file(slot, i) (at most capacity
    // bytes); its length follows it to the host (read_lens) on s: the file length, or when it exceeds capacity the length it
    // needs (nothing past capacity is written), or that needed length's lower bound | kJpegLenLowerBound.  Returns the
    // number of kernels launched.
    int encode(int n, const JpegSrc &src, int components, int w, int h, int quality, size_t capacity, int slot, cudaStream_t s);
    const FileSlots &files() const { return files_; }
    // The exact length image i of src needs, given a length reported over capacity; synchronises s.  A lower bound is
    // resolved by encoding the image alone in a workspace and files of its own, so encodes of this encoder still in flight
    // on other streams (the next group of a pipeline) are neither read nor overwritten.
    size_t needed(uint64_t reported, const JpegSrc &src, int i, int components, int w, int h, int quality, cudaStream_t s);

  private:
    int encode_part(int n, const JpegSrc &src, int components, int w, int h, int quality, size_t capacity, uint8_t *files,
                    uint64_t *lens, cudaStream_t s);
    DeviceBuffer<uint8_t> ws_;
    FileSlots files_;
    std::unique_ptr<JpegExactEncoder> probe_;  // needed()'s own encoder, created on first use
};

}  // namespace dfb
