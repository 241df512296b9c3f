// block_scan.cuh — CTA-wide exclusive scan and sum, shared by the PNG and JPEG encoders.
#pragma once

#include <cuda_runtime.h>

namespace dfb {

// exclusive scan over the CTA; *total receives the sum.  sm: NT / 32 words.
template <int NT, typename T> __device__ T block_scan(T v, T &total, T *sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sm[warp] = x;
    __syncthreads();
    if (warp == 0) {
        T t = lane < NT / 32 ? sm[lane] : T(0);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        if (lane < NT / 32) sm[lane] = t;
    }
    __syncthreads();
    const T base = warp ? sm[warp - 1] : T(0);
    total = sm[NT / 32 - 1];
    __syncthreads();
    return base + x - v;
}

template <int NT, typename T> __device__ T block_sum(T v, T *sm) {
    T total;
    block_scan<NT>(v, total, sm);
    return total;
}

}  // namespace dfb
