// Layout of a batch's scratch regions inside one device buffer (QueryCtx::d_cand / d_lab).  Host C++ only.
//
// A layout is written once, as a function of the base that takes its regions from a BatchScratch, and run twice: over a null
// base to size it (bytes()), then over the buffer grown to that size to bind its pointers.  Both passes take the same regions
// in the same order, so they agree.  Take the pointers after the last grow of that buffer: growing reallocates it.
#pragma once
#include <cstddef>
#include <cstdint>

namespace rsb200 {

class BatchScratch {
  public:
    // Every region starts at a multiple of 256 bytes from `base`, which cudaMalloc aligns to 256: enough for 16-byte vector
    // access and TMA.
    static constexpr size_t kAlign = 256;

    explicit BatchScratch(void *base = nullptr) : base_(static_cast<uint8_t *>(base)) {}

    // the next `count` elements of T; nullptr for count == 0 (no space used) and in the sizing pass
    template <class T> T *take(size_t count) {
        if (count == 0) return nullptr;
        used_ = (used_ + kAlign - 1) / kAlign * kAlign;
        T *p = base_ ? reinterpret_cast<T *>(base_ + used_) : nullptr;
        used_ += count * sizeof(T);
        return p;
    }
    size_t bytes() const { return used_; }
    size_t words() const { return (used_ + 7) / 8; } // in uint64_t elements, as QueryCtx::need_cand / need_lab take it

  private:
    uint8_t *base_;
    size_t used_ = 0;
};

} // namespace rsb200
