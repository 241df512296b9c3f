// png_encode.h — imencode(".png", img) of packed 8-bit BGR images on the GPU, byte-identical to OpenCV's default PNG
// parameters (filter SUB, zlib level 1, strategy Z_RLE, libpng's 8 KB IDAT chunks).  See png_encode.cu.
#pragma once

#include "file_slots.h"

namespace dfb {

// upper bound of the file size of a w x h image (every deflate block stored, plus headers and chunk framing)
size_t png_max_bytes(int w, int h);

// Workspace and output files of the encoder, grown on demand.
class PngEncoder {
  public:
    PngEncoder() = default;
    PngEncoder(const PngEncoder &) = delete;
    PngEncoder &operator=(const PngEncoder &) = delete;
    // Encodes n images of w x h enqueued on s: image i's rows start at src + i * img_stride, bgr_pitch bytes apart.  File i
    // is written to files().file(slot, i); its length (0: the encoder failed) follows it to the host (read_lens) on s.
    // Returns the number of kernels launched.
    int encode(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, int slot, cudaStream_t s);
    const FileSlots &files() const { return files_; }

  private:
    int encode_part(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, uint8_t *files, uint64_t *lens,
                    cudaStream_t s);
    DeviceBuffer<uint8_t> ws_;  // per-image workspace, see png_encode.cu
    FileSlots files_;
};

}  // namespace dfb
