// png_pack.h — convertFlowToPngImage on the GPU (/root/reference/src/common.cpp:18-46), see png_pack.cu.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace dfb {

struct PngBounds {
    double bound_x, bound_y;            // after the "+4 when divisible by 8" rule
    float min_x, max_x, min_y, max_y;   // minMaxLoc of the two components
};

constexpr int kPngPackBlocks = 528;  // 4 x 132 SMs

size_t png_pack_scratch_bytes();
// flow_xy: CV_32FC2 rows (pitch in bytes); bgr: packed 3 bytes per pixel (pitch in bytes).  scratch: png_pack_scratch_bytes()
// of device memory, zero-initialised once.  *bounds_dev receives the device address of the bounds this launch computes.
void launch_flow_to_png_image(const float *flow_xy, size_t flow_pitch_bytes, int w, int h, uint8_t *bgr, size_t bgr_pitch, void *scratch,
                              PngBounds **bounds_dev, cudaStream_t s);

}  // namespace dfb
