// tma.cuh — sm_90a bulk-tensor (TMA) + mbarrier helpers shared by the stencil kernels: cp.async.bulk.tensor.2d loads of
// fp32 tiles into shared memory (zero fill outside the tensor), completion on an mbarrier, and the host-side descriptor
// encoder (cuTensorMapEncodeTiled through the runtime's driver entry point: the library does not link libcuda).
#pragma once

#include <cuda_runtime.h>

namespace dfb {

constexpr int kTensorMapBytes = 128;  // sizeof(CUtensorMap)

// Encodes one 2-D fp32 tile descriptor (box box_w x box_h elements, no swizzle, zero fill out of bounds) into out[128 bytes].
// plane: base pointer (16-byte aligned), extent w x h (elements / rows), row pitch in elements (a multiple of 4).
// box_w * 4 must be a multiple of 16 bytes; both box edges <= 256.
void encode_tensor_map_2d(void *out, const float *plane, int w, int h, int pitch, int box_w, int box_h);

#ifdef __CUDACC__
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 2-D tile load global -> shared, completion signalled on the mbarrier (zero fill outside the tensor; x, y may be negative)
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const void *tmap, int x, int y, unsigned long long *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar))
                 : "memory");
}
// Asks the TMA unit to bring a tile into L2 only (no shared-memory destination, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_l2_2d(const void *tmap, int x, int y) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// generic-proxy accesses to shared memory before this fence are ordered before later async-proxy (TMA) writes to it
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// global memory written through the generic proxy (plain stores, by this or — after a barrier this thread has observed — by
// other CTAs) is ordered before the async-proxy (TMA) reads this thread issues afterwards
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
#endif

}  // namespace dfb
