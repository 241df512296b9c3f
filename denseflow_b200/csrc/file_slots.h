// file_slots.h — the output files of a batch encoder, in two slots so the read-back of one group can overlap the encode of
// the next.  Per slot: n files of at most file_cap bytes and their lengths, on the device and (pinned) on the host.
#pragma once

#include <stdexcept>
#include <string>

#include "common.cuh"

namespace dfb {

class FileSlots {
  public:
    // room for n files of at most file_cap bytes in `slot`
    void prepare(int slot, int n, size_t file_cap) {
        Slot &S = slots_[slot];
        S.file_cap = file_cap;
        S.files.grow((size_t)n * file_cap);
        S.lens.grow(sizeof(uint64_t) * n);
        S.host_lens.grow(sizeof(uint64_t) * n);
    }
    uint8_t *file(int slot, int i) const { return slots_[slot].files + (size_t)i * slots_[slot].file_cap; }
    uint64_t *lens(int slot) const { return slots_[slot].lens; }
    // enqueues the copy of the slot's first n lengths to the host on s
    void read_lens(int slot, int n, cudaStream_t s) const {
        DFB_CUDA(cudaMemcpyAsync(slots_[slot].host_lens, slots_[slot].lens, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost, s));
    }
    // length k of the slot once read_lens has completed
    uint64_t host_len(int slot, int k) const { return slots_[slot].host_lens[k]; }
    // After read_lens(slot, n, ·) has completed.  In file order, a length of 0 (no file) or over capacity fails the call with
    // std::runtime_error(reject(k, length)) for the first such file k.  Then file k is copied to out(k, length) on s, the bytes
    // are added to d2h_bytes and s is synchronised.
    template <typename Reject, typename Out>
    void deliver(int slot, int n, size_t capacity, Reject &&reject, Out &&out, uint64_t &d2h_bytes, cudaStream_t s) const {
        const uint64_t *lens = slots_[slot].host_lens;
        for (int k = 0; k < n; ++k)
            if (lens[k] == 0 || lens[k] > capacity) throw std::runtime_error(reject(k, lens[k]));
        for (int k = 0; k < n; ++k) {
            const size_t len = (size_t)lens[k];
            DFB_CUDA(cudaMemcpyAsync(out(k, len), file(slot, k), len, cudaMemcpyDeviceToHost, s));
            d2h_bytes += len;
        }
        DFB_CUDA(cudaStreamSynchronize(s));
    }

  private:
    struct Slot {
        DeviceBuffer<uint8_t> files;
        DeviceBuffer<uint64_t> lens;
        PinnedBuffer<uint64_t> host_lens;
        size_t file_cap = 0;
    };
    Slot slots_[2];
};

}  // namespace dfb
