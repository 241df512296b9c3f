// common.cuh — shared helpers for the sm_90a flow engine (device planes, error plumbing).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

namespace dfb {

// fp32 image plane in HBM. pitch is in ELEMENTS and always a multiple of 32 (128-byte rows): every
// row starts on a cache line, float4 accesses never straddle a row end, and the stride satisfies
// TMA's 16-byte rule. Columns [w, pitch) are padding: kernels may write garbage there and never
// let it reach a valid pixel (all border rules are predicated on image coordinates).
struct Plane {
    float *p;
    int w, h, pitch;
};

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

struct CudaError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

inline void check(cudaError_t e, const char *what, const char *file, int line) {
    if (e != cudaSuccess) {
        throw CudaError(std::string(what) + ": " + cudaGetErrorString(e) + " (" + file + ":" + std::to_string(line) + ")");
    }
}
#define DFB_CUDA(x) ::dfb::check((x), #x, __FILE__, __LINE__)
#define DFB_KERNEL_CHECK() ::dfb::check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__)

// The error of a call without a handle: dfb_last_error(NULL) reports msg afterwards (dfb_api.cu).  Returns code.
int fail_unbound(int code, const std::string &msg);

// convertFlowToImage, /root/reference/src/common.cpp:4-16: the CAST macro evaluates in double (the bounds are double),
// left to right, then cvRound (round-half-to-even).  Shared by the stand-alone quantiser and the merge epilogues.
#ifdef __CUDACC__
__device__ __forceinline__ uint8_t quantise_px(float v, double L, double H) {
    if ((double)v > H) return 255;
    if ((double)v < L) return 0;
    const double q = 255 * ((double)v - L) / (H - L);
    if (q != q) return 0;
    return (uint8_t)__double2int_rn(q);
}
#endif

// Bump allocator over one cudaMalloc slab: all engine workspace is carved out at create time
// (no allocation ever happens on the per-pair path).
class Slab {
  public:
    Slab() = default;
    ~Slab() { release(); }
    Slab(const Slab &) = delete;
    Slab &operator=(const Slab &) = delete;
    void reserve(size_t bytes) {
        release();
        DFB_CUDA(cudaMalloc(&base_, bytes));
        cap_ = bytes;
        off_ = 0;
    }
    void release() {
        if (base_) cudaFree(base_);
        base_ = nullptr;
        cap_ = off_ = 0;
    }
    template <typename T> T *take(size_t n) {
        size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
        if (off_ + bytes > cap_) throw std::runtime_error("dfb: workspace slab exhausted");
        T *r = reinterpret_cast<T *>(static_cast<char *>(base_) + off_);
        off_ += bytes;
        return r;
    }
    static size_t padded(size_t n, size_t elem) { return (n * elem + 255) & ~size_t(255); }
    size_t used() const { return off_; }
    void zero() { if (base_) DFB_CUDA(cudaMemset(base_, 0, cap_)); }

  private:
    void *base_ = nullptr;
    size_t cap_ = 0, off_ = 0;
};

// One owned allocation of device memory (Pinned = false: cudaMalloc) or page-locked host memory (true: cudaHostAlloc),
// sized in bytes and freed by the destructor.
template <typename T, bool Pinned> class OwnedBuffer {
  public:
    OwnedBuffer() = default;
    ~OwnedBuffer() { release(); }
    OwnedBuffer(const OwnedBuffer &) = delete;
    OwnedBuffer &operator=(const OwnedBuffer &) = delete;
    // Room for at least `bytes`.  Work on any stream may still use the old buffer, so the device is synchronised first.
    void grow(size_t bytes) {
        if (bytes <= cap_) return;
        DFB_CUDA(cudaDeviceSynchronize());
        allocate(bytes);
    }
    // The same without the synchronisation: for a first allocation, or when the caller has waited for the buffer's last user.
    void allocate(size_t bytes) {
        if (bytes <= cap_) return;
        release();
        void *p = nullptr;
        DFB_CUDA(Pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes));
        p_ = static_cast<T *>(p);
        cap_ = bytes;
    }
    operator T *() const { return p_; }
    size_t bytes() const { return cap_; }

  private:
    void release() {
        if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
    }
    T *p_ = nullptr;
    size_t cap_ = 0;
};
template <typename T> using DeviceBuffer = OwnedBuffer<T, false>;
template <typename T> using PinnedBuffer = OwnedBuffer<T, true>;

}  // namespace dfb
