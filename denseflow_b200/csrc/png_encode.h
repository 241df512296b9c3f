// png_encode.h — imencode(".png", img) of packed 8-bit BGR images on the GPU, byte-identical to OpenCV's default PNG
// parameters (filter SUB, zlib level 1, strategy Z_RLE, libpng's 8 KB IDAT chunks).  See png_encode.cu.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dfb {

// upper bound of the file size of a w x h image (every deflate block stored, plus headers and chunk framing)
size_t png_max_bytes(int w, int h);

// Workspace and output files of the encoder, grown on demand.  Files live in two slots so the read-back of one batch can
// overlap the encode of the next.
class PngEncoder {
  public:
    PngEncoder() = default;
    PngEncoder(const PngEncoder &) = delete;
    PngEncoder &operator=(const PngEncoder &) = delete;
    ~PngEncoder();
    // Encodes n images of w x h enqueued on s: image i's rows start at src + i * img_stride, bgr_pitch bytes apart.  File i
    // is written to file(slot, i), its length to lens(slot)[i] (device memory).  Returns the number of kernels launched.
    int encode(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, int slot, cudaStream_t s);
    const uint8_t *file(int slot, int i) const { return files_[slot] + (size_t)i * file_cap_; }
    uint64_t *lens(int slot) const { return lens_[slot]; }

  private:
    void ensure(int n, int w, int h, int slot);
    int encode_part(int n, const uint8_t *src, size_t img_stride, size_t bgr_pitch, int w, int h, uint8_t *files, uint64_t *lens,
                    cudaStream_t s);
    uint8_t *ws_ = nullptr;  // per-image workspace, see png_encode.cu
    size_t ws_cap_ = 0;
    uint8_t *files_[2] = {};
    size_t files_cap_[2] = {};
    uint64_t *lens_[2] = {};
    int lens_n_[2] = {};
    size_t file_cap_ = 0;
};

}  // namespace dfb
