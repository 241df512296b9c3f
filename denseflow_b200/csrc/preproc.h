// preproc.h — BGR->gray and INTER_LINEAR uint8 resize, bit-exact to OpenCV's CPU path (see preproc.cu).
#pragma once

#include <vector>

#include "common.cuh"

namespace dfb {

struct ResizeTap {
    int idx;     // first source index (unclamped for rows)
    int a0, a1;  // 11-bit fixed-point weights of idx and idx + 1
};

void build_resize_taps(int dn, int sn, bool reset_at_borders, std::vector<ResizeTap> &out);
void launch_bgr_to_gray(const uint8_t *bgr, size_t bgr_pitch, int w, int h, uint8_t *gray, size_t gray_pitch, cudaStream_t s);
void launch_resize_u8(const uint8_t *src, size_t src_pitch, int sw, int sh, uint8_t *dst, size_t dst_pitch, int dw, int dh,
                      const ResizeTap *xt, const ResizeTap *yt, cudaStream_t s);
// Packed BGR (sw x sh) -> INTER_LINEAR resize to dw x dh (xt == yt == nullptr: no resize, sw == dw and sh == dh) -> libjpeg's
// JFIF YCbCr -> 4:2:0.  y: dw x dh; cb, cr: c_cols x ceil(dh / 2), sharing c_pitch, where c_cols = 0 means ceil(dw / 2).
// Wider chroma rows are the compressor's padded extent: the columns past ceil(dw / 2) are downsampled from the replicated
// last full-resolution column, as libjpeg's expand_right_edge leaves them (jpeg_chroma_cols, jpeg_encode.h).
void launch_bgr_to_ycc420(const uint8_t *bgr, size_t bgr_pitch, int sw, int sh, int dw, int dh, const ResizeTap *xt, const ResizeTap *yt,
                          uint8_t *y, size_t y_pitch, uint8_t *cb, uint8_t *cr, size_t c_pitch, cudaStream_t s, int c_cols = 0);

}  // namespace dfb
