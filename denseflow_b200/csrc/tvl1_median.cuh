// tvl1_median.cuh — the optional k x k median of the flow between TV-L1 iterations (DESIGN §4.3), k = 3 or 5: one
// definition for the fused pair kernel, its stage hook and the stand-alone kernel of the unfused schedule.
//
// M_k(u) at a pixel is the element of rank (k*k - 1) / 2, in ascending order with -0 below +0, of the k x k window with
// index-clamped (replicate) borders.  A median selects one of its inputs, so every build computes it exactly.
#pragma once

#include <climits>
#include <utility>

#include "common.cuh"

namespace dfb {

// Floats as signed integers in a total order: ascending value, -0 below +0.  Every exchange of the network is an integer
// min / max of these keys, so the result, the sign of a zero included, does not depend on how min.f32 / max.f32 order
// signed zeros.  The map is its own inverse.
__device__ __forceinline__ int median_key(float v) {
    const int b = __float_as_int(v);
    return b ^ ((b >> 31) & 0x7fffffff);
}
__device__ __forceinline__ float median_value(int key) { return __int_as_float(key ^ ((key >> 31) & 0x7fffffff)); }

// Batcher's odd-even merge sort of N keys (N a power of two) as a list of exchanges (lo, hi), built at compile time.
struct MedianNet {
    int n;
    unsigned char lo[192], hi[192];
};
template <int N>
__host__ __device__ constexpr MedianNet median_net() {
    MedianNet c{};
    for (int p = 1; p < N; p <<= 1)
        for (int k = p; k >= 1; k >>= 1)
            for (int j = k % p; j + k < N; j += 2 * k)
                for (int i = 0; i < k && i + j + k < N; ++i)
                    if ((i + j) / (2 * p) == (i + j + k) / (2 * p)) {
                        c.lo[c.n] = (unsigned char)(i + j);
                        c.hi[c.n] = (unsigned char)(i + j + k);
                        ++c.n;
                    }
    return c;
}
// Every exchange with constant indices, so the keys stay in registers.  Only the exchanges the middle element depends on
// survive dead-code elimination, and those against the INT_MAX padding fold away.
template <int N, int... C>
__device__ __forceinline__ void median_sort(int (&a)[N], std::integer_sequence<int, C...>) {
    constexpr MedianNet net = median_net<N>();
    static_assert(net.n <= 192, "network fits its table");
    auto exchange = [&](int i, int j) {
        const int lo = min(a[i], a[j]), hi = max(a[i], a[j]);
        a[i] = lo;
        a[j] = hi;
    };
    (exchange(net.lo[C], net.hi[C]), ...);
}

// The median of the K x K window whose top-left element is s[0] (row pitch sp floats, shared memory).
template <int K>
__device__ __forceinline__ float median_window(const float *s, int sp) {
    constexpr int N = K * K <= 16 ? 16 : 32;
    int a[N];
#pragma unroll
    for (int dy = 0; dy < K; ++dy)
#pragma unroll
        for (int dx = 0; dx < K; ++dx) a[dy * K + dx] = median_key(s[dy * sp + dx]);
#pragma unroll
    for (int i = K * K; i < N; ++i) a[i] = INT_MAX;
    median_sort(a, std::make_integer_sequence<int, median_net<N>().n>());
    return median_value(a[(K * K - 1) / 2]);
}

constexpr int kMedianHalo = 2;  // staged border: enough for k = 5
constexpr int kMedianTileW = 32;
template <int NT>
struct MedianTile {
    static constexpr int TH = NT / 32;                          // output rows per tile (one pixel per thread)
    static constexpr int SW = kMedianTileW + 2 * kMedianHalo;   // staged row pitch
    static constexpr int SH = TH + 2 * kMedianHalo;
    static constexpr int kStage = SW * SH;                      // floats of shared memory per plane
};

// dst = M_k(src) for u1 and u2 of a W x H level (row pitch P floats), run by NT threads of every block of a grid-stride
// loop over 32 x NT/32 tiles (block bid of nblocks).  Both planes of a tile are staged into shared memory (s1, s2:
// MedianTile<NT>::kStage floats each) with index-clamped reads, then every thread writes one pixel of each.  Only the
// W x H image pixels of dst are written.  The sources are read through L2 (__ldcg): other blocks wrote them.  The caller
// synchronises the block before it reuses s1 / s2.
template <int NT>
__device__ __forceinline__ void median_planes(const float *u1, const float *u2, float *d1, float *d2, int W, int H, int P, int k, int bid,
                                              int nblocks, float *s1, float *s2) {
    using T = MedianTile<NT>;
    const int ntx = (W + kMedianTileW - 1) / kMedianTileW, nty = (H + T::TH - 1) / T::TH;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int t = bid; t < ntx * nty; t += nblocks) {
        const int y0 = (t / ntx) * T::TH, x0 = (t % ntx) * kMedianTileW;
        __syncthreads();  // the previous tile's windows have been read
        for (int i = threadIdx.x; i < T::kStage; i += NT) {
            const int sy = i / T::SW, sx = i - sy * T::SW;
            const size_t o = (size_t)min(max(y0 + sy - kMedianHalo, 0), H - 1) * P + min(max(x0 + sx - kMedianHalo, 0), W - 1);
            s1[i] = __ldcg(u1 + o);
            s2[i] = __ldcg(u2 + o);
        }
        __syncthreads();
        const int x = x0 + tx, y = y0 + ty;
        if (x < W && y < H) {
            const int r = k >> 1;
            const int so = (ty + kMedianHalo - r) * T::SW + tx + kMedianHalo - r;
            const size_t o = (size_t)y * P + x;
            if (k == 3) {
                d1[o] = median_window<3>(s1 + so, T::SW);
                d2[o] = median_window<3>(s2 + so, T::SW);
            } else {
                d1[o] = median_window<5>(s1 + so, T::SW);
                d2[o] = median_window<5>(s2 + so, T::SW);
            }
        }
    }
}

}  // namespace dfb
