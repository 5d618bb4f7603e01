// Device-side building blocks shared by the KNN scan kernels and the BM25 top-N kernel:
// order-preserving keys, a per-warp streaming top-k list in shared memory, and an in-smem
// bitonic sort.  All selection is done on ONE unsigned 64-bit composite per candidate:
//
//     composite = (orderable_key(score) << 32) | internal_row_id
//
// so "k best" is "k smallest composites": total order, NaN-safe, deterministic.  This reproduces
// the reference's heap ordering — a max-heap of pair<float,size_t> under std::less
// (VS/utils/vecsim_stl.h:64-84) fed in ascending internal-id order with a strict `<` admission
// test (VS/algorithms/brute_force/brute_force.h:272-278): among equal scores the earliest ids
// survive, exactly what (score,id) lexicographic selection yields.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace rsb200 {

constexpr uint64_t kEmptySlot = 0xFFFFFFFFFFFFFFFFull; // sorts after every real candidate
constexpr uint32_t kNaNKey = 0xFFFFFFFEu;              // NaN distances sort after +inf
constexpr int kMaxFusedK = 128;                        // largest k the fused per-warp lists take
constexpr int kMaxWideK = 1024;                        // largest k of a batch on the device (chunks of kMaxFusedK beyond it)

// float -> uint32 whose unsigned order equals the float order (-inf < ... < -0 == +0 < ... < +inf
// < NaN).
__device__ __forceinline__ uint32_t orderable_key(float x) {
    if (x != x) return kNaNKey;
    uint32_t u = __float_as_uint(x + 0.0f); // -0 -> +0
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __host__ __forceinline__ float key_to_float(uint32_t key) {
    if (key >= 0xFFFFFFFEu) {
        uint32_t nanbits = 0x7FC00000u;
#ifdef __CUDA_ARCH__
        return __uint_as_float(nanbits);
#else
        float f;
        memcpy(&f, &nanbits, 4);
        return f;
#endif
    }
    uint32_t u = (key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
__device__ __forceinline__ uint64_t make_composite(float score, uint32_t id) {
    return ((uint64_t)orderable_key(score) << 32) | id;
}

__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int mask) {
    uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, mask);
    uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), mask);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)v, src);
    uint32_t hi = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}

// A k-entry unsorted list owned by one warp, living in shared memory.  `worst` (the largest
// composite in the list, i.e. the admission threshold) and `worst_pos` are warp-uniform registers.
// Admission is rare after warm-up (expected k*ln(rows/k) per warp), so the replace+rescan cost is
// irrelevant next to the scan itself.
struct WarpTopK {
    uint64_t *slots; // [k] in shared memory
    uint32_t k;
    uint64_t worst;
    uint32_t worst_pos;

    __device__ __forceinline__ void init(uint64_t *smem_slots, uint32_t k_, int lane) {
        slots = smem_slots;
        k = k_;
        for (uint32_t p = lane; p < k; p += 32) slots[p] = kEmptySlot;
        worst = kEmptySlot;
        worst_pos = 0;
        __syncwarp();
    }
    // Warp-uniform candidate; must be called by all 32 lanes.
    __device__ __forceinline__ void admit(uint64_t cand, int lane) {
        if (lane == 0) slots[worst_pos] = cand;
        __syncwarp();
        uint64_t best = 0;
        uint32_t pos = 0;
        for (uint32_t p = lane; p < k; p += 32) {
            uint64_t v = slots[p];
            if (v >= best) { // >= so that a list full of equal values still yields a valid pos
                best = v;
                pos = p;
            }
        }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
            uint64_t ob = shfl_xor_u64(best, m);
            uint32_t op = __shfl_xor_sync(0xffffffffu, pos, m);
            if (ob > best || (ob == best && op < pos)) {
                best = ob;
                pos = op;
            }
        }
        worst = best;
        worst_pos = pos;
    }
    // Each lane may hold its own candidate (valid==false -> nothing to offer).  Lanes whose
    // candidate beats the threshold are admitted one after the other in lane order.
    __device__ __forceinline__ void offer(bool valid, uint64_t cand, int lane) {
        unsigned pending = __ballot_sync(0xffffffffu, valid && cand < worst);
        while (pending) {
            int src = __ffs(pending) - 1;
            pending &= pending - 1;
            uint64_t c = shfl_u64(cand, src);
            if (c < worst) admit(c, lane); // threshold may have tightened since the ballot
        }
    }
};

// Ascending bitonic sort of n (power of two) composites in shared memory by one CTA.
__device__ __forceinline__ void bitonic_sort_smem(uint64_t *buf, uint32_t n) {
    for (uint32_t size = 2; size <= n; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (uint32_t t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                uint32_t lo = 2 * t - (t & (stride - 1));
                uint32_t hi = lo + stride;
                bool up = ((lo & size) == 0);
                uint64_t a = buf[lo], b = buf[hi];
                if ((a > b) == up) {
                    buf[lo] = b;
                    buf[hi] = a;
                }
            }
        }
    }
    __syncthreads();
}

__host__ __device__ __forceinline__ uint32_t next_pow2(uint32_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

} // namespace rsb200
