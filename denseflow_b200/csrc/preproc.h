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
// How much of the planes launch_bgr_to_ycc420 writes, with cw = ceil(dw / 2) and ch = ceil(dh / 2):
//   image        y: dw x dh, cb / cr: cw x ch
//   chroma_cols  y: dw x dh, cb / cr: round8(cw) x ch (what JpegExactEncoder reads: jpeg_chroma_cols, jpeg_encode.h)
//   mcu          y: round16(dw) x round16(dh), cb / cr: round8(cw) x round8(ch) (whole MCUs, what nvJPEG reads)
// Padding is libjpeg's: luma columns and rows past the image repeat its last column and row; chroma columns past cw are
// downsampled from the replicated last full-resolution column (expand_right_edge, jcsample.c) and chroma rows past ch repeat
// the last chroma row (expand_bottom_edge, jcprepct.c).
enum class YccExtent { image, chroma_cols, mcu };
// Packed BGR (sw x sh) -> INTER_LINEAR resize to dw x dh (xt == yt == nullptr: no resize, sw == dw and sh == dh) -> libjpeg's
// JFIF YCbCr -> 4:2:0 planes y (y_pitch) and cb, cr (sharing c_pitch), over `extent`.
void launch_bgr_to_ycc420(const uint8_t *bgr, size_t bgr_pitch, int sw, int sh, int dw, int dh, const ResizeTap *xt, const ResizeTap *yt,
                          uint8_t *y, size_t y_pitch, uint8_t *cb, uint8_t *cr, size_t c_pitch, cudaStream_t s,
                          YccExtent extent = YccExtent::image);
// Replicates the last column and row of n w x h gray planes (pitch bytes, plane_stride apart) in place up to pw x ph.
void launch_pad_edges(uint8_t *planes, size_t pitch, size_t plane_stride, int n, int w, int h, int pw, int ph, cudaStream_t s);

}  // namespace dfb
