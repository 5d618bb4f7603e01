// Batched KNN on the tensor cores (wgmma, sm_90a).  Replaces, for query batches, the B independent passes of
// BruteForceIndex::topKQuery (VS/algorithms/brute_force/brute_force.h:243-291) + the distance kernels of VS/spaces/.
//
// fp32 cosine corpora — coarse-then-exact (DESIGN.md §4): 256 queries x 10M x 768 is 3.93 TFLOP per corpus pass,
// FMA-bound on CUDA cores, and no tensor-core operand type reproduces the reference's fp32 bits.  So
//   stage 1  a wgmma GEMM with APPROXIMATE distances keeps, per CTA row range and query, the kCoarseKeep best rows
//            (coarse_wgmma_kernel<false,...> over an fp16 shadow copy, or coarse_kernel<CfgTF32> over the fp32 rows);
//   stage 2  rescore_kernel recomputes those candidates from the fp32 rows with the bit-exact arithmetic of
//            distance_core.cuh;
//   stage 3  verify_kernel proves per query that no discarded row can belong to the exact top-k — otherwise the query
//            falls back to the exact scan, on the device.
// fp16 / bf16 corpora (coarse_wgmma_kernel<true,*,0>) and int8 / uint8 corpora (<true,*,1|2>, s8 / u8 wgmma): the
// tensor-core result IS the distance (16-bit: fp32-accumulated exact products, bar 1e-2; 8-bit: exact integer dot
// products + the reference's float expression, bit-exact), each CTA keeps its exact top-k.
//
// coarse_wgmma_kernel (one CTA per SM, persistent over the 128-row tiles of its row range):
//   warp 0    producer: row tiles into an n-stage shared-memory ring (contiguous bulk copies from the tiled shadow, or
//             128B-swizzle tensor-map boxes from a row-major 16/8-bit corpus), multicast across the query-group cluster
//   warps 4-7 one warpgroup: wgmma m64n128 (M = the CTA's 64 queries, resident in shared memory for the whole pass;
//             N = 128 rows of the ring stage; 32 bytes of K per instruction), register accumulators, then the
//             epilogue: the accumulators are transposed through shared memory so that a thread owns one query, raw
//             dot products are tested against a register threshold, survivors go to a per-query list in global memory
//             that a warp-wide radix select cuts back to the best `keep`.  The fixed-bound pass tests its bound on the
//             accumulator fragment itself (no transpose) and appends survivors at slots from shared per-query counters;
//             it runs a second such warpgroup (warps 8-11), the two taking the CTA's tiles alternately so that one's
//             drain and bound test overlap the other's MMAs.
// coarse_kernel<CfgTF32>: the SS shape with the rows as the M operand (32 queries per CTA in shared memory), kept for
// fp32 corpora without shadow memory (mode 2) and rows too wide for the 16-bit kernel's shared memory.
#include "coarse_tc.h"
#include "distance_core.cuh"
#include "topk_common.cuh"

#include <cuda.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <type_traits>

namespace rsb200 {

constexpr int kTileM = 128;       // rows per tile of coarse_kernel (two m64 wgmma blocks)
constexpr int kMaxStages = 8;     // ring depth is chosen at plan time from the shared memory left over
constexpr int kCoarseThreads = 256;
constexpr int kListCap = 64;      // per-query candidate buffer in shared memory
constexpr uint32_t kStageBytes = kTileM * 128; // one K block of a row tile: 128 rows x 128 bytes = 16 KB
constexpr int kTF32StageStride = 33;           // coarse_kernel accumulator transpose: [128 rows][33 words]

struct CfgTF32 {
    static constexpr int kTileN = 32;   // queries per CTA (wgmma N)
    static constexpr int kBlockK = 32;  // elements per K block = 128 bytes = one swizzle row
    static constexpr int kElem = 4;
};

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// one lane of a converged warp; keeps the surrounding code warp-uniform so that barrier addresses stay in uniform
// registers
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred;
    asm volatile(
        "{\n"
        ".reg .pred P;\n"
        "elect.sync _|P, 0xffffffff;\n"
        "selp.b32 %0, 1, 0, P;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or the hint expires)
// instead of spinning, which leaves issue slots to the warps doing the work
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
            : "memory");
    } while (!done);
}
// pure spin (no suspend hint): for the waits whose wake-up latency is on the critical path (the producer and the
// warpgroup that issues the MMAs)
__device__ __forceinline__ void mbar_wait_spin(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// slice of a tile delivered to the same shared-memory offset of every CTA in `mask`
__device__ __forceinline__ void tma_load_2d_mc(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
// contiguous global -> shared copy through the TMA engine (no tensor map), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// the same, delivered to the same shared-memory offset of every CTA in `mask`; each destination's mbarrier (same
// offset) receives the byte count
__device__ __forceinline__ void bulk_load_1d_mc(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
        : "memory");
}
// pull `bytes` of global memory into L2 ahead of a later bulk copy (no completion to wait for)
__device__ __forceinline__ void bulk_prefetch_l2(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
// address of `local_smem_addr` in the shared memory of CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
    return r;
}
// arrive on an mbarrier of another CTA of the cluster.  Default semantics (release at CTA scope), which compile to the
// arrive alone: a release at cluster scope adds a GPU-wide memory barrier before every arrive.  The ring stages this
// releases are read only by wgmma (the async proxy), and those reads are complete once wgmma.wait_group has returned,
// so there is no generic-proxy access for a cluster-scope release to order before the producer's refill.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire;" ::: "memory");
}

// ---- wgmma (one warpgroup, both operands in shared memory, register accumulators) ----------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving reads of the accumulators above the wait that makes them valid
template <class T, int N>
__device__ __forceinline__ void wg_fence_operands(T (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) {
        if constexpr (sizeof(T) == 4 && std::is_same<T, float>::value)
            asm volatile("" : "+f"(d[i])::"memory");
        else
            asm volatile("" : "+r"(d[i])::"memory");
    }
}
// D (+)= A * B^T, A = 64 rows (M) and B = 128 rows (N) of K-major 128B-swizzled tiles; 32 bytes of K per instruction
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// the same with A from registers: this thread's fragment of the 64 x 16 A tile, (row r, halves c, c + 1) per register,
// a = {(r0, c0), (r0 + 8, c0), (r0, c0 + 8), (r0 + 8, c0 + 8)} with r0 = 16 (warp % 4) + lane / 4, c0 = 2 (lane % 4)
__device__ __forceinline__ void wgmma_f16_n128_ra(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_s8_n128(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_u8_n128(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// the m64n128 wgmma of an operand type: kInt = 8-bit (kVar 1 = int8, else uint8), else 16-bit (kVar 1 = bf16, else fp16)
template <bool kInt, int kVar, class Acc>
__device__ __forceinline__ void wgmma_n128(Acc (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (kInt && kVar == 1)
        wgmma_s8_n128(d, adesc, bdesc, scale_d);
    else if constexpr (kInt)
        wgmma_u8_n128(d, adesc, bdesc, scale_d);
    else if constexpr (kVar == 1)
        wgmma_bf16_n128(d, adesc, bdesc, scale_d);
    else
        wgmma_f16_n128(d, adesc, bdesc, scale_d);
}

// K-major, 128B-swizzled operand tile: rows of 128 bytes, 8-row groups 1024 bytes apart.  wgmma matrix descriptor:
// start>>4 [0,14), leading byte offset>>4 [16,30) (unused for swizzled K-major: 1), stride byte offset>>4 [32,46),
// layout type [62,64) = 1 (SWIZZLE_128B).  Advancing the start by 32 bytes (+2) steps K inside the swizzled row.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ------------------------------------------------------------------------------------------------
// TF32 on the fp32 rows: rows are the M operand (128 per tile = two m64 blocks), the CTA's 32 queries the N operand.
// Warps 4-7 (one warpgroup) issue the MMAs, transpose the accumulators through shared memory so that a thread owns one
// row of the tile, and run the candidate-list epilogue.
// ------------------------------------------------------------------------------------------------
template <class Cfg>
__global__ void __launch_bounds__(kCoarseThreads, 1)
coarse_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_q, uint32_t n_rows, uint32_t nq,
              uint32_t num_kb, uint32_t tiles_total, uint32_t keep, uint32_t nstages, uint64_t *__restrict__ cand_out) {
    constexpr int kTileN = Cfg::kTileN;
    constexpr int kHalves = kTileN / 32;
    constexpr uint32_t kQBlockBytes = kTileN * 128;
    static_assert(kTileN == 32, "the accumulator transpose assumes 32 queries per CTA");
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *sQ = smem;                                   // num_kb x [kTileN x 128B]
    uint8_t *sA = sQ + (size_t)num_kb * kQBlockBytes;     // nstages x [128 x 128B]
    uint32_t *sacc = reinterpret_cast<uint32_t *>(sA + (size_t)nstages * kStageBytes); // [128 rows][kTF32StageStride]
    uint64_t *lists = reinterpret_cast<uint64_t *>(sacc + kTileM * kTF32StageStride);  // [kTileN][kListCap]
    uint64_t *bars = lists + kTileN * kListCap;
    uint64_t *full = bars, *empty = bars + kMaxStages;
    uint64_t *qbar = empty + kMaxStages;
    uint32_t *counts = reinterpret_cast<uint32_t *>(qbar + 1); // [kTileN]
    uint32_t *thresh = counts + kTileN;                        // [kTileN] orderable keys
    uint32_t *pending_flag = thresh + kTileN;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t q_base = blockIdx.y * kTileN;
    // this CTA's tiles: t = blockIdx.x, blockIdx.x + gridDim.x, ...
    const uint32_t my_tiles = (tiles_total > blockIdx.x) ? (tiles_total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < nstages; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_init(qbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        *pending_flag = 0;
    }
    if (threadIdx.x < kTileN) {
        counts[threadIdx.x] = 0;
        thresh[threadIdx.x] = 0xFFFFFFFFu;
    }
    __syncthreads();

    if (warp == 0) {
        // ===== TMA producer =====
        if (elect_one_sync()) {
            mbar_expect_tx(qbar, num_kb * kQBlockBytes);
            for (uint32_t kb = 0; kb < num_kb; kb++)
                tma_load_2d(sQ + (size_t)kb * kQBlockBytes, &map_q, qbar, (int)(kb * Cfg::kBlockK), (int)q_base);
        }
        __syncwarp();
        uint32_t s = 0, ph = 0;
        for (uint32_t i = 0; i < my_tiles; i++) {
            const uint32_t tile = blockIdx.x + i * gridDim.x;
            for (uint32_t kb = 0; kb < num_kb; kb++) {
                mbar_wait(&empty[s], ph ^ 1);
                if (elect_one_sync()) {
                    mbar_expect_tx(&full[s], kStageBytes);
                    tma_load_2d(sA + (size_t)s * kStageBytes, &map_a, &full[s], (int)(kb * Cfg::kBlockK), (int)(tile * kTileM));
                }
                __syncwarp();
                if (++s == nstages) s = 0, ph ^= 1;
            }
        }
    } else if (warp >= 4) {
        // ===== MMA + epilogue: accumulators -> shared memory -> registers -> candidate lists =====
        const int ew = warp - 4;                 // warp of the warpgroup: accumulator rows 16 ew .. 16 ew + 15 of each m64 block
        const int et = threadIdx.x - 128;        // 0..127 = row of the tile in the epilogue
        mbar_wait(qbar, 0);
        uint32_t s = 0, ph = 0;
        const uint64_t bdesc_first = make_smem_desc(smem_u32(sQ));
        constexpr uint64_t kQStep = kQBlockBytes >> 4, kHalfTile = (kStageBytes / 2) >> 4;
        for (uint32_t i = 0; i < my_tiles; i++) {
            const uint32_t tile = blockIdx.x + i * gridDim.x;
            float acc[2][16];
            uint32_t prev = 0;
            for (uint32_t kb = 0; kb < num_kb; kb++) {
                mbar_wait_spin(&full[s], ph);
                wg_fence(); // the accumulator registers are handed to the MMA pipe for this stage's run
                const uint64_t ad = make_smem_desc(smem_u32(sA + (size_t)s * kStageBytes));
                const uint64_t bd = bdesc_first + (uint64_t)kb * kQStep;
#pragma unroll
                for (int kk = 0; kk < 4; kk++) { // 8 tf32 = 32 bytes of K per instruction
                    const uint32_t acc_on = (kb | (uint32_t)kk) != 0;
                    wgmma_tf32_n32(acc[0], ad + 2 * kk, bd + 2 * kk, acc_on);
                    wgmma_tf32_n32(acc[1], ad + kHalfTile + 2 * kk, bd + 2 * kk, acc_on);
                }
                wg_commit();
                wg_wait<1>(); // the previous stage's MMAs have retired (nothing to wait for on the first): its slot may be refilled
                if (kb != 0 && et == 0) mbar_arrive(&empty[prev]);
                prev = s;
                if (++s == nstages) s = 0, ph ^= 1;
            }
            wg_wait<0>();
            if (et == 0) mbar_arrive(&empty[prev]);
            wg_fence_operands(acc[0]);
            wg_fence_operands(acc[1]);
            // accumulator fragment: acc[mb][4j + 2 i2 + c] = (row 64 mb + 16 ew + lane / 4 + 8 i2, query 8 j + 2 (lane % 4) + c)
            asm volatile("bar.sync 1, 128;" ::: "memory"); // the previous tile's reads of sacc are done
#pragma unroll
            for (int mb = 0; mb < 2; mb++)
#pragma unroll
                for (int j = 0; j < 4; j++)
#pragma unroll
                    for (int x = 0; x < 4; x++) {
                        const int r = 64 * mb + 16 * ew + (lane >> 2) + 8 * (x >> 1), c = 8 * j + 2 * (lane & 3) + (x & 1);
                        sacc[r * kTF32StageStride + c] = __float_as_uint(acc[mb][4 * j + x]);
                    }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            uint32_t v[kHalves][32];
#pragma unroll
            for (int h = 0; h < kHalves; h++)
#pragma unroll
                for (int j = 0; j < 32; j++) v[h][j] = sacc[et * kTF32StageStride + h * 32 + j];
            const uint32_t row = tile * kTileM + et;
            uint32_t pend[kHalves]; // bit j: candidate for query h*32+j still to be stored
#pragma unroll
            for (int h = 0; h < kHalves; h++) {
                pend[h] = 0;
                if (row < n_rows) {
#pragma unroll
                    for (int j = 0; j < 32; j++) {
                        const float d = 1.0f - __uint_as_float(v[h][j]);
                        v[h][j] = orderable_key(d);
                        if (v[h][j] < thresh[h * 32 + j]) pend[h] |= 1u << j;
                    }
                }
            }
            // insert with retry: lists are compacted (keep best `keep`) whenever they run full
            for (;;) {
                uint32_t any_left = 0;
#pragma unroll
                for (int h = 0; h < kHalves; h++) {
                    uint32_t still = 0;
                    uint32_t p = pend[h];
                    while (p) {
                        const int jj = __ffs(p) - 1;
                        p &= p - 1;
                        uint32_t key = 0;
#pragma unroll
                        for (int x = 0; x < 32; x++)
                            if (x == jj) key = v[h][x];
                        const int j = h * 32 + jj;
                        if (key >= thresh[j]) continue; // threshold tightened meanwhile
                        const uint32_t slot = atomicAdd(&counts[j], 1u);
                        if (slot < (uint32_t)kListCap)
                            lists[j * kListCap + slot] = ((uint64_t)key << 32) | row;
                        else
                            still |= 1u << jj;
                    }
                    pend[h] = still;
                    any_left |= still;
                }
                if (any_left) *pending_flag = 1;
                asm volatile("bar.sync 1, 128;" ::: "memory");
                // compaction: warp ew handles queries j = ew, ew+4, ...
                const uint32_t any_pending = *pending_flag;
                for (int j = ew; j < kTileN; j += 4) {
                    const uint32_t c = min(counts[j], (uint32_t)kListCap);
                    if (c < (uint32_t)(kListCap / 2) && !any_pending) continue;
                    if (c <= keep) {
                        if (lane == 0) counts[j] = c;
                        continue;
                    }
                    // each lane holds up to 2 entries; extract the `keep` smallest by repeated warp-min
                    uint64_t e0 = (lane < (int)c) ? lists[j * kListCap + lane] : kEmptySlot;
                    uint64_t e1 = (lane + 32 < (int)c) ? lists[j * kListCap + lane + 32] : kEmptySlot;
                    __syncwarp();
                    uint64_t last = 0;
                    for (uint32_t r = 0; r < keep; r++) {
                        uint64_t m = e0 < e1 ? e0 : e1;
#pragma unroll
                        for (int sft = 16; sft > 0; sft >>= 1) {
                            const uint64_t o = shfl_xor_u64(m, sft);
                            m = o < m ? o : m;
                        }
                        if (e0 == m) e0 = kEmptySlot; else if (e1 == m) e1 = kEmptySlot;
                        if (lane == 0) lists[j * kListCap + r] = m;
                        last = m;
                    }
                    if (lane == 0) {
                        counts[j] = keep;
                        thresh[j] = (uint32_t)(last >> 32);
                    }
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");
                if (!any_pending) break;
                if (et == 0) *pending_flag = 0;
                asm volatile("bar.sync 1, 128;" ::: "memory");
            }
        }
        // final compaction + publish: cand_out[q][blockIdx.x][keep]
        asm volatile("bar.sync 1, 128;" ::: "memory");
        for (int j = ew; j < kTileN; j += 4) {
            const uint32_t c = min(counts[j], (uint32_t)kListCap);
            uint64_t e0 = (lane < (int)c) ? lists[j * kListCap + lane] : kEmptySlot;
            uint64_t e1 = (lane + 32 < (int)c) ? lists[j * kListCap + lane + 32] : kEmptySlot;
            const uint32_t q = q_base + j;
            for (uint32_t r = 0; r < keep; r++) {
                uint64_t m = e0 < e1 ? e0 : e1;
#pragma unroll
                for (int sft = 16; sft > 0; sft >>= 1) {
                    const uint64_t o = shfl_xor_u64(m, sft);
                    m = o < m ? o : m;
                }
                if (e0 == m) e0 = kEmptySlot; else if (e1 == m) e1 = kEmptySlot;
                if (lane == 0 && q < nq) cand_out[((size_t)q * gridDim.x + blockIdx.x) * keep + r] = m;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// 16-bit / 8-bit operands with the QUERIES as the M operand and the rows as N (M = 64 queries, N = 128 rows per
// wgmma).  The 64 queries of a CTA are written once into shared memory (swizzled like the row tiles) and stay there for
// the whole pass; the ring only carries the streaming row tiles.  One warpgroup issues the MMAs of a tile (register
// accumulators, 64 per thread), then transposes them through shared memory so that in the epilogue a thread owns one
// QUERY: its threshold lives in a register and its candidate list needs no atomics.  64 queries per CTA (not 128) so
// that the resident queries fit shared memory next to the ring up to 1024 dimensions (16 KB per 128 dimensions per 128
// queries would leave no room for the ring at 768); threads 64-127 of the warpgroup take part in the MMAs and the
// warp-wide selections but own no query.  The fixed-bound pass over the int8 shadow, whose queries take half the bytes,
// holds 128 (coarse_cta_queries).
//   The candidate lists live in global memory (L2): appends are rare once the thresholds have settled, and shared
//   memory goes to the row-tile ring.
// ------------------------------------------------------------------------------------------------
constexpr int kQM = 64;             // queries per CTA (wgmma M)
constexpr int kQN = 128;            // rows per tile = N of one wgmma
constexpr int kQMaxStages = 16;
constexpr int kQKbPerStage = 2;     // K blocks per pipeline stage: amortises the barrier round trip over 8 MMAs.  The K block
                                    // count is padded to a multiple of it (coarse_kb: zero blocks), so every stage is the same
                                    // straight run of MMAs and the compiler never has to reconcile two MMA sequences
// candidate lists: kEpl entries per lane of the compacting warp -> kEpl*32 slots per query; a list is cut back to
// `keep` when it holds more than (slots - 32) entries after a 32-row chunk.  kEpl = 3 (96 slots) serves keep <= 32,
// kEpl = 8 (256 slots) keep <= 128.
constexpr int kQListStride = 129;   // lists[slot * stride + query slot]: conflict-free appends
constexpr uint32_t kQBlockBytes = kQN * 128;                    // one K block of a row tile: 128 rows x 128 bytes
constexpr uint32_t kQStageBytes = kQKbPerStage * kQBlockBytes; // 32 KB
// K blocks of `bytes_per_row` bytes of operand (128 per block), padded to whole stages: the padding blocks are zero in the
// queries (and in the fp16 shadow; tensor-map loads past the row fill zeros), so they add nothing to the dot products
__host__ __device__ constexpr uint32_t coarse_kb(uint32_t bytes_per_row) {
    return ((bytes_per_row + 127) / 128 + kQKbPerStage - 1) / kQKbPerStage * kQKbPerStage;
}
constexpr int kQAccStride = kQN + 4;                            // accumulator transpose [64 queries][132 words]
constexpr uint32_t kQAccBytes = kQM * kQAccStride * 4;
// The fixed-bound pass (mode 1) runs two consumer warpgroups that take the CTA's tiles alternately: one warpgroup's
// drain and bound test run under the other's MMAs instead of leaving the tensor pipe idle at every tile boundary
// (DESIGN.md §4.2: 5,022 -> 4,294 clk per tile at 10M x 768).  The sample pass over the int8 shadow (kOp 5, mode 2) runs
// two as well, on the wide CTA below: its epilogue reads the accumulator fragment too.  The other modes keep one: their
// epilogue transposes through shared memory and compacts lists, which a second warpgroup would have to double.
// The passes whose epilogue works on the accumulator fragment in registers (no transpose buffer)
__host__ __device__ constexpr bool coarse_frag_epilogue(bool q8, int mode) { return mode == 1 || (q8 && mode == 2); }
__host__ __device__ constexpr int coarse_consumers(bool q8, int mode) { return coarse_frag_epilogue(q8, mode) ? 2 : 1; }
// Queries per CTA.  The fixed-bound and sample passes over the int8 shadow (kOp 5, modes 1 and 2) hold 128: each consumer
// warpgroup owns 64 of them and both run their MMAs against every ring stage, so a row tile is copied into shared memory once
// per 128 queries instead of once per 64 (384 instead of 480 KB of shared-memory traffic per 128 queries x 128 rows, DESIGN.md
// §4.2), and at a batch of 256 the two query groups of a row range form clusters of two, which fill all the SMs.  Its int8
// queries take 128 B per K block and query, so 128 of them leave at least three ring stages up to 1024 dimensions
__host__ __device__ constexpr int coarse_cta_queries(bool q8, int mode) { return q8 && (mode == 1 || mode == 2) ? 2 * kQM : kQM; }
// warp 0 produces, warps 1-3 idle, warps 4.. are the consumer warpgroups
__host__ __device__ constexpr int coarse_threads(bool q8, int mode) { return 128 * (1 + coarse_consumers(q8, mode)); }

// bar.sync / bar.arrive on a named barrier (ids 1-3 in coarse_wgmma_kernel; 0 is __syncthreads)
template <int kId, int kCount>
__device__ __forceinline__ void named_sync() {
    asm volatile("bar.sync %0, %1;" ::"n"(kId), "n"(kCount) : "memory");
}
template <int kId, int kCount>
__device__ __forceinline__ void named_arrive() {
    asm volatile("bar.arrive %0, %1;" ::"n"(kId), "n"(kCount) : "memory");
}

// Cycle account of the fixed-bound pass (tools/coarse_cycles.py), compiled only with -DCOARSE_CYCLE_ACCOUNT: per CTA and
// role (consumer warpgroup 0, 1, producer), clock64() sums of the phases below.  Without the macro every call is empty
// and the kernels compile to the same code as without the calls.
enum : int { kCaPass, kCaWait, kCaIssue, kCaWait1, kCaEpilogue, kCaHandoff, kCaTiles, kCaSlots };
#ifdef COARSE_CYCLE_ACCOUNT
constexpr int kCaMaxCtas = 1024;
__device__ unsigned long long g_coarse_cycles[kCaMaxCtas][3][kCaSlots];
struct CycleAccount {
    unsigned long long v[kCaSlots] = {};
    __device__ __forceinline__ long long now() const { return clock64(); }
    __device__ __forceinline__ void add(int slot, long long t0) { v[slot] += (unsigned long long)(clock64() - t0); }
    __device__ __forceinline__ void count(int slot) { v[slot]++; }
    __device__ __forceinline__ void flush(uint32_t cta, int role) {
        if (cta < (uint32_t)kCaMaxCtas)
            for (int i = 0; i < kCaSlots; i++) g_coarse_cycles[cta][role][i] = v[i];
    }
};
#else
struct CycleAccount {
    __device__ __forceinline__ long long now() const { return 0; }
    __device__ __forceinline__ void add(int, long long) {}
    __device__ __forceinline__ void count(int) {}
    __device__ __forceinline__ void flush(uint32_t, int) {}
};
#endif

// Cut list `q` (c entries, keep < c <= 32 * kEpl) back to its `keep` smallest, unordered, in slots [0, keep); returns the
// key of the worst kept entry (the new admission threshold).  Warp-wide radix select on the 32-bit key — 32 rounds
// of ballots — instead of `keep` rounds of warp-min extraction (measured: 21K clk per call, a third of the
// epilogue's time and, worse, a stall of the accumulator hand-back).  Among entries tied with the threshold key the
// lowest row ids are kept, so the kept set is exactly the `keep` smallest composites (key, row).
template <int kEpl>
__device__ __forceinline__ uint32_t select_keep(uint64_t *lists, int q, uint32_t c, uint32_t keep, int lane) {
    __syncwarp(); // the list was appended to by one lane: order its (global-memory) writes before the warp's reads
    uint64_t e[kEpl];
    uint32_t k[kEpl];
    bool v[kEpl];
#pragma unroll
    for (int t = 0; t < kEpl; t++) {
        const uint32_t idx = lane + 32 * t;
        v[t] = idx < c;
        e[t] = v[t] ? lists[idx * kQListStride + q] : kEmptySlot;
        k[t] = (uint32_t)(e[t] >> 32);
    }
    __syncwarp();
    uint32_t prefix = 0, remaining = keep;
#pragma unroll 1
    for (int bit = 31; bit >= 0; bit--) {
        const uint32_t hi_mask = bit == 31 ? 0u : ~((2u << bit) - 1u); // the bits already decided
        uint32_t zeros = 0;
#pragma unroll
        for (int t = 0; t < kEpl; t++) {
            const bool z = v[t] && ((k[t] ^ prefix) & hi_mask) == 0 && !((k[t] >> bit) & 1u);
            zeros += __popc(__ballot_sync(0xFFFFFFFFu, z));
        }
        if (zeros < remaining) {
            remaining -= zeros;
            prefix |= 1u << bit;
        }
    }
    // prefix = keep-th smallest key; `remaining` (>= 1) entries equal to it are still needed
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t base = 0;
#pragma unroll
    for (int t = 0; t < kEpl; t++) {
        const bool less = v[t] && k[t] < prefix;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, less);
        if (less) lists[(base + __popc(m & lt)) * kQListStride + q] = e[t];
        base += __popc(m);
    }
    // entries tied with the threshold key: the `remaining` LOWEST row ids stay (the exact scan admits rows in id order
    // with a strict `<`), found by a second radix select on the low word when there are more ties than places
    uint32_t n_eq = 0;
#pragma unroll
    for (int t = 0; t < kEpl; t++) n_eq += __popc(__ballot_sync(0xFFFFFFFFu, v[t] && k[t] == prefix));
    uint32_t row_cut = 0xFFFFFFFFu; // keep tied entries with row <= row_cut
    if (n_eq > remaining) {
        uint32_t rp = 0, rem = remaining;
#pragma unroll 1
        for (int bit = 31; bit >= 0; bit--) {
            const uint32_t hi_mask = bit == 31 ? 0u : ~((2u << bit) - 1u);
            uint32_t zeros = 0;
#pragma unroll
            for (int t = 0; t < kEpl; t++) {
                const uint32_t row = (uint32_t)e[t];
                const bool z = v[t] && k[t] == prefix && ((row ^ rp) & hi_mask) == 0 && !((row >> bit) & 1u);
                zeros += __popc(__ballot_sync(0xFFFFFFFFu, z));
            }
            if (zeros < rem) {
                rem -= zeros;
                rp |= 1u << bit;
            }
        }
        row_cut = rp; // row ids are unique: exactly `remaining` tied entries have row <= rp
    }
#pragma unroll
    for (int t = 0; t < kEpl; t++) {
        const bool eq = v[t] && k[t] == prefix && (uint32_t)e[t] <= row_cut;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, eq);
        if (eq) lists[(base + __popc(m & lt)) * kQListStride + q] = e[t];
        base += __popc(m);
    }
    __syncwarp();
    return prefix;
}

// Fixed-radius pass over 8-bit corpora: the largest integer x with (float)x <= r, the pre-test bound of the integer distances
// (1 - dot for inner product, the int32 e of L2).  int -> float rounding is monotone, so {x : (float)x <= r} is the set of
// integers up to that x and `x <= range_int_bound(r)` is exactly `(float)x <= r` for |x| < 2^30 (8-bit distances stay below
// 2^29).  floor(r) is in the set (below 2^24 it is exact; above, r is itself an integer); the loop adds the integers above r
// that round down to it (at most half an ulp of r, 64 at 2^30).  NaN: nothing passes; beyond +-2^30: everything / nothing.
__device__ __forceinline__ int range_int_bound(float r) {
    if (!(r == r) || r < -1073741824.0f) return INT_MIN;
    if (r >= 1073741824.0f) return INT_MAX;
    int x = (int)floorf(r);
    while (__int2float_rn(x + 1) <= r) x++;
    return x;
}

// int8 shadow (kOp 5): an integer bound ti with  fl(sqt * a) > tdot  =>  a > ti  for every int32 accumulator a (|a| < 2^24,
// exact in float), sqt = fl(s_q s_t), so that `a > ti` never drops a row the float test keeps.  No division: rq = fl(1 / s_q) is
// taken once per query and rt = fl(1 / s_t) once per tile, and f = fl(tdot fl(rq rt)) is tdot / sqt up to six roundings of
// 2^-24 relative (rq, rt, their product and f; sqt and fl(sqt a) on the test's side), under 3.6e-7 in all, which the 1e-5
// relative loosening covers many times over; one more integer covers the rounding of the loosening and a subnormal f.  The
// argument needs fl(rq rt) in [2^-125, 2^125], which keeps s_q s_t normal: outside it, and for NaN, everything passes.  A bound
// beyond +-2^25: everything / nothing.
__device__ __forceinline__ int q8_dot_bound(float tdot, float rq, float rt) {
    const float r = __fmul_rn(rq, rt);
    const float f = __fmul_rn(tdot, r);
    if (!(f == f) || !(r >= 0x1p-125f && r <= 0x1p125f)) return INT_MIN;
    const float c = fminf(fmaxf(f, -33554432.0f), 33554432.0f);
    return (int)floorf(c - fabsf(c) * 1e-5f) - 1;
}

// kDirect = false: fp32 corpus, rows come from the tiled fp16 shadow (bulk copies), output = sorted candidate lists for
//                  the exact rescoring + proof.
// kDirect = true : fp16 / bf16 corpus, rows come straight from the row-major corpus through a 128B-swizzle tensor
//                  map; the fp32-accumulated products of the stored 16-bit values ARE the distances (the reference's
//                  own tiers differ by more: SURVEY.md finding 5, bar 1e-2), so each CTA keeps its exact top-`keep`
//                  and the lists go to final_select unsorted.
//   kOp = 0  16-bit float operands, fp32 accumulators: distance 1 - dot
//   kOp = 1  int8 / uint8 operands (s8 / u8 wgmma), int32 accumulators, inner product: (float)(1 - dot)  (IP.cpp:248-252)
//   kOp = 2  the same, cosine: 1 - (float)dot / (norm_row * norm_query), norms = the fp32 stored after the payload
//            (IP.cpp:264-271).  The integer dot products are exact, so kOp 1/2 reproduce the reference bit for bit.
//   kOp = 3  16-bit float operands, squared L2 from the GEMM: (|q|^2 + |row|^2) - 2 dot, with the squared norms of
//            the fp32 rows / queries in row_norm2 / q_norm2 (coarse stage of the fp32 L2 route)
//   kOp = 4  int8 / uint8 operands, squared L2: (float)(|row|^2 + |q|^2 - 2 dot) evaluated in int32, with the exact int32
//            squared norms in row_norm2 / q_norm2 (the pointers carry int32).  The integer is the reference's exact sum
//            (L2.cpp:148-174), rounded once to float as it is, so kOp 4 is bit-exact too.  Each term is at most
//            65025 * dim <= 1.4e8 at the widest 8-bit dim (2048): no int32 overflow.
//   kFixed   the admission threshold of every query is FIXED for the whole pass (thr_fixed[q], a distance, from the sample
//            pass): every row with approximate distance < thr_fixed[q] is kept — no running threshold, no list compaction;
//            a list that runs full sets overflow[q] (the query goes to the next tier).  fp32 route (kOp 0 / 3) and 16-bit
//            corpora.  8-bit corpora (kOp 1 / 2 / 4): thr_fixed[q] is the radius of a range query and a row is kept iff its
//            exact float distance d satisfies d <= thr_fixed[q] (range_int_bound for the pre-tests, DESIGN.md §4.11).
//            list_count (nullable): list_count[q][blockIdx.x] = the entries of the published list (min(appends, keep)).
//            The int8 shadow's pass (kOp 5) needs it and publishes only those entries, without the kEmptySlot padding:
//            refine_kernel, its one reader, reads the counts.  Every other fixed pass pads its lists.
//   kSample  the sample pass: no lists at all — per (query, row range) the smallest approximate distance of each of
//            kCoarseSampleSlices = 32 disjoint slices of the range's sampled rows (32-row chunk of the tile x tile counter
//            mod 8), published as keep = 32 composites.  Over the int8 shadow the slices follow the accumulator fragment
//            instead: row 8 j + 2 (lane % 4) + c of the tile falls in slice (lane % 4, c, tile counter mod 4), so that every
//            thread keeps its minima in registers.  Each minimum is the approximate distance of a distinct sampled row, so
//            the k-th smallest of a query's lists x 32 minima is an upper bound of its k-th best distance over the sample (k
//            distinct rows are at or below it), which is all the fixed bound needs.
//   tile_stride > 1: only every tile_stride-th row tile is visited (the sample pass)
//   kVar     operand type: 16-bit operands 1 = bfloat16 (else IEEE half); 8-bit 1 = int8 (else uint8).  A template parameter so
//            that the MMA sequence of a stage is one straight run of wgmma instructions (no branch between them)
//   kFilt    hybrid batches (DESIGN.md §4.10): only rows whose bit is set in the query's row-space bitmap count.  Query q's
//            bitmap is filt + filt_words * (filt_q ? filt_q[q] : q).  The sample pass takes each chunk's maximum over its
//            filtered rows; the adaptive lists and the fixed bound admit only filtered rows (the fixed bound tests the bit on
//            its rare survivor path, after the key test).  fp32 route, and the 8-bit fixed-radius pass (DESIGN.md §4.13), which
//            tests the bit after both the integer pre-test and the float range test.
//   kOp = 5  the int8 shadow of unit fp32 rows (s8 wgmma, int32 accumulators): the approximate distance is
//            1 - fl(fl(s_q s_t) acc), s_q = the query's scale (a float after its int8 payload), s_t = the row tile's scale
//            (row_norm2[tile]).  The fixed-bound pass tests one integer bound per (query, tile) on the accumulators; the sample
//            and adaptive-list passes turn the accumulators into those float dot products in the transpose and then run kOp 0's
//            epilogue.  Unit vectors only; the error bound is per query (DESIGN.md §4.2)
//   kRegKb   the fixed-bound pass over the fp16 shadow: the first kRegKb K blocks of the CTA's queries are held in registers
//            (the wgmma A fragment, 16 per K block and thread, loaded once per consumer warpgroup) instead of shared memory,
//            which frees kRegKb x 8 KB for the ring (DESIGN.md §4.2).  The first kRegKb / kQKbPerStage stages of a tile take
//            A from those registers; the MMA sequence in K is unchanged, so every distance is the same.  0 = all in sQ.
template <bool kDirect, int kEpl, int kOp, int kMode, int kVar = 0, bool kFilt = false, int kRegKb = 0>
__global__ void __launch_bounds__(coarse_threads(kOp == 5, kMode), 1)
coarse_wgmma_kernel(const __grid_constant__ CUtensorMap map_rows, const uint8_t *__restrict__ shadow, size_t row_pitch,
                    const uint8_t *__restrict__ q16, size_t q16_pitch, const float *__restrict__ row_norm2,
                    const float *__restrict__ q_norm2, uint32_t n_rows, uint32_t nq, uint32_t dim, uint32_t row_bytes,
                    uint32_t num_kb, uint32_t tiles_total, uint32_t keep, uint32_t nstages, uint32_t csize,
                    uint64_t *__restrict__ list_scratch, uint64_t *__restrict__ cand_out, const uint32_t *__restrict__ nq_dev,
                    uint32_t tile_stride, const float *__restrict__ thr_fixed, uint32_t *__restrict__ overflow,
                    const uint32_t *__restrict__ filt, uint32_t filt_words, const uint32_t *__restrict__ filt_q,
                    uint32_t *__restrict__ list_count) {
    constexpr bool kFixed = kMode == 1, kSample = kMode == 2;
    constexpr bool kQ8 = kOp == 5;
    constexpr bool kInt = kOp == 1 || kOp == 2 || kOp == 4 || kQ8;
    constexpr int kOpE = kQ8 ? 0 : kOp; // the epilogue of kOp 5 past the integer bound test is kOp 0's
    constexpr bool kFrag = coarse_frag_epilogue(kQ8, kMode); // no transpose buffer
    constexpr int kCons = coarse_consumers(kQ8, kMode), kConsThreads = 128 * kCons;
    // kWide: 128 queries per CTA, warpgroup cw takes the MMAs and the epilogue of queries 64 cw .. 64 cw + 63 of every tile
    constexpr int kCtaQ = coarse_cta_queries(kQ8, kMode);
    constexpr bool kWide = kCtaQ > kQM;
    static_assert(!kWide || (kCons == 2 && kCtaQ == kCons * kQM), "a wide CTA: one consumer warpgroup per 64 queries");
    constexpr uint32_t kQKbBytes = kCtaQ * 128; // one K block of the resident queries
    using Acc = typename std::conditional<kInt, uint32_t, float>::type;
    // bx = row range, by = query group
    const uint32_t bx = blockIdx.x, by = blockIdx.y, gx = gridDim.x;
    static_assert(kMode == 0 || (!kDirect && (kOp == 0 || kOp == 3 || kQ8)) || (kDirect && kOp == 0) || (kDirect && kFixed && kInt && kEpl == 8),
                  "fixed bound / sample pass: the fp32 route and 16-bit corpora (inner product / cosine); fixed radius: 8-bit corpora");
    static_assert(!kQ8 || (!kDirect && !kFilt && kRegKb == 0 && kVar == 1), "int8 shadow: signed operands, no filters");
    static_assert(!kFilt || (!kDirect && (kOp == 0 || kOp == 3)) || (kDirect && kFixed && kInt && kEpl == 8),
                  "row filters: the fp32 route and the 8-bit fixed-radius pass");
    static_assert(kRegKb == 0 || (!kDirect && kFixed && kRegKb % kQKbPerStage == 0),
                  "register-held queries: the fixed-bound pass over the fp16 shadow, whole stages");
    // kFilt: the row-space bitmap of the query at position `pos` of this batch
    auto filt_row = [&](uint32_t pos) { return filt + (size_t)filt_words * (filt_q ? filt_q[pos] : pos); };
    // the sample's slices: tiles i, i + kSliceSets, ... share a slice set of 4 chunks of 32 rows per tile.  kFrag: the slices
    // (lane % 4, c, h) of the accumulator fragment, 4 x 2 x 4 (kSliceSets = 4 is then the number of 32-row chunks h)
    constexpr int kSliceSets = (int)kCoarseSampleSlices / (kFrag ? 8 : kQN / 32);
    static_assert(!kSample || kSliceSets * (kFrag ? 8 : kQN / 32) == (int)kCoarseSampleSlices, "whole slice sets");
    static_assert(!(kSample && kFrag) || kSliceSets == kQN / 32, "kFrag: a slice per 32-row chunk and (lane % 4, c)");
    constexpr int kQListCap = kEpl * 32;
    if (nq_dev) { // second tier: the number of live queries is only known on the device; nothing to do = every CTA leaves
        nq = min(nq, *nq_dev);
        if (nq == 0) return;
    }
    constexpr uint32_t kQTrigger = kQListCap - 32;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms, by an offset of smem_raw itself: the pointers stay visibly shared,
    // so their accesses compile to STS / LDS rather than generic stores and loads
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *sB = smem;                                                   // nstages x kQKbPerStage x [128 rows x 128B]
    // K blocks kRegKb .. num_kb - 1 x [64 queries x 128B], swizzled; kWide: two such 64-query halves per K block
    uint8_t *sQ = sB + (size_t)nstages * kQStageBytes;
    uint32_t *sacc = reinterpret_cast<uint32_t *>(sQ + (size_t)(num_kb - kRegKb) * kQKbBytes); // [kQM][kQAccStride]; not kFrag
    uint64_t *bars = reinterpret_cast<uint64_t *>(sacc + (kFrag ? 0 : kQM * kQAccStride));
    uint64_t *full = bars, *empty = bars + kQMaxStages;
    uint32_t *qcount = reinterpret_cast<uint32_t *>(bars + 2 * kQMaxStages); // kFixed: [kCtaQ] appends per query
    // this CTA's candidate lists [kQListCap][kQListStride]
    uint64_t *lists = list_scratch + (size_t)(by * gx + bx) * (kQListCap * kQListStride);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t q_base = by * kCtaQ;
    const uint32_t my_tiles = (tiles_total > bx) ? (tiles_total - bx + gx - 1) / gx : 0;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < nstages; s++) {
            mbar_init(&full[s], 1);
            // multicast clusters: every CTA of the cluster reads the stage and releases it (kWide: each of its warpgroups)
            mbar_init(&empty[s], kWide ? kCons * csize : csize);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    // cluster mode: the csize CTAs that share blockIdx.x (one per query group) walk the SAME row tiles.
    // Each fetches 1/csize of every stage and multicasts it into all csize shared memories, so a tile leaves
    // HBM/L2 once per cluster instead of once per query group.
    const uint32_t crank = (csize > 1) ? cluster_ctarank() : 0;
    const uint16_t cmask = (uint16_t)((1u << csize) - 1u);
    if (csize > 1) cluster_sync_all(); // peers must see initialised barriers before anything is signalled remotely

    CycleAccount ca;
    const uint32_t cta = by * gx + bx;
    if (warp == 0) {
        // ===== producer: row tiles [128 rows x 128 bytes] per K block, kQKbPerStage K blocks per stage =====
        uint32_t s = 0, ph = 0;
        const uint32_t slice = kQStageBytes / csize; // num_kb is a multiple of kQKbPerStage: every stage is full
        const long long t_pass = ca.now();
        for (uint32_t i = 0; i < my_tiles; i++) {
            const uint32_t tile = (bx + i * gx) * tile_stride;
            ca.count(kCaTiles);
            for (uint32_t kb0 = 0; kb0 < num_kb; kb0 += kQKbPerStage) {
                const uint32_t kbn = min((uint32_t)kQKbPerStage, num_kb - kb0);
                const long long t_wait = ca.now();
                mbar_wait_spin(&empty[s], ph ^ 1);
                ca.add(kCaWait, t_wait);
                if (elect_one_sync()) {
                    const uint32_t bytes = kbn * kQBlockBytes;
                    mbar_expect_tx(&full[s], bytes);
                    if constexpr (kDirect) {
                        // row-major 16/8-bit corpus: one 128B-swizzle box of (128 / csize) rows x 128 bytes per K block
                        const uint32_t slice_rows = kQN / csize;
                        for (uint32_t j = 0; j < kbn; j++) {
                            uint8_t *dst = sB + (size_t)s * kQStageBytes + j * kQBlockBytes + crank * slice_rows * 128;
                            const int c0 = (int)((kb0 + j) * ((kOp == 0 || kOp == 3) ? 64 : 128)), c1 = (int)(tile * kQN + crank * slice_rows);
                            if (csize > 1)
                                tma_load_2d_mc(dst, &map_rows, &full[s], c0, c1, cmask);
                            else
                                tma_load_2d(dst, &map_rows, &full[s], c0, c1);
                        }
                    } else {
                        // the shadow copy is stored tile by tile in the swizzled shared-memory image (to_f16_tiled_kernel):
                        // the K blocks of a stage are one contiguous run in HBM
                        const uint8_t *src = shadow + ((size_t)tile * num_kb + kb0) * kQBlockBytes;
                        // fixed-bound pass: the same slice of the CTA's next tile into L2, so that its bulk copy waits on L2
                        // rather than HBM.  Only two of the ring's stages can load ahead of the MMAs, which is too little
                        // to cover HBM latency (DESIGN.md §4.2); one tile ahead is 5.8 MB of L2 at 10M x 768, four thrash it.
                        // The int8 sample pass likewise, its next tile tile_stride x gx tiles on
                        if constexpr (kFixed || (kSample && kFrag)) {
                            const size_t ahead = (size_t)gx * (kFixed ? 1u : tile_stride) * num_kb * kQBlockBytes;
                            if (i + 1 < my_tiles) bulk_prefetch_l2(src + ahead + crank * slice, slice);
                        }
                        if (csize > 1) {
                            bulk_load_1d_mc(sB + (size_t)s * kQStageBytes + crank * slice, src + crank * slice, slice, &full[s], cmask);
                        } else {
                            bulk_load_1d(sB + (size_t)s * kQStageBytes, src, bytes, &full[s]);
                        }
                    }
                }
                __syncwarp();
                if (++s == nstages) s = 0, ph ^= 1;
            }
        }
        ca.add(kCaPass, t_pass);
        if (kFixed && lane == 0) ca.flush(cta, 2);
    } else if (warp >= 4) {
        const int cw = kCons > 1 ? (warp - 4) >> 2 : 0; // consumer warpgroup (0 .. kCons - 1)
        const int ew = kCons > 1 ? (warp - 4) & 3 : warp - 4; // warp of the warpgroup: accumulator rows (queries) 16 ew .. 16 ew + 15
        // 0..127 within the warpgroup; the query slot in the epilogue (slots >= kQM own no query)
        const int et = kCons > 1 ? (threadIdx.x - 128) & 127 : threadIdx.x - 128;
        // kWide: the CTA's query slots of this warpgroup start at wq, its queries at qw
        const int wq = kWide ? kQM * cw : 0;
        const uint32_t qw = q_base + wq;
        const uint32_t q = qw + et;
        const bool live = et < kQM && q < nq;
        // ===== queries -> shared memory (zero padded to num_kb * 128 bytes and to kCtaQ queries) =====
        if ((kWide || cw == 0) && et < kQM) {
            const uint4 *src = reinterpret_cast<const uint4 *>(q16 + (size_t)q * q16_pitch);
            for (uint32_t kb = kRegKb; kb < num_kb; kb++) {
                // row `et` of a K-major 128B-swizzled operand tile: chunk u at et*128 + ((u ^ (et & 7)) * 16)
                uint8_t *row = sQ + (size_t)(kb - kRegKb) * kQKbBytes + wq * 128 + et * 128;
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    uint4 x = make_uint4(0, 0, 0, 0);
                    if (live && kb * 128 + u * 16 < row_bytes) x = src[kb * 8 + u];
                    *reinterpret_cast<uint4 *>(row + ((u ^ (et & 7)) * 16)) = x;
                }
            }
            if constexpr (kFixed) qcount[wq + et] = 0;
        }
        // kRegKb: this thread's A fragments of K blocks 0 .. kRegKb - 1 (k16 step t = 4 kb + kk), straight from q16 in every
        // consumer warpgroup, zero padded as sQ is (query slots >= nq, bytes past the row).  The wgmma.fence in front of
        // each stage's MMAs orders these register writes before the first MMA that reads them.
        uint32_t qa[kRegKb ? 4 * kRegKb : 1][4];
        if constexpr (kRegKb > 0) {
#pragma unroll
            for (int i2 = 0; i2 < 2; i2++) {
                const uint32_t fq = qw + 16 * ew + (lane >> 2) + 8 * i2;
                const uint8_t *src = q16 + (size_t)fq * q16_pitch;
#pragma unroll
                for (int t = 0; t < 4 * kRegKb; t++)
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint32_t off = 32 * t + 4 * (lane & 3) + 16 * h; // halves 16 t + 2 (lane % 4) + 8 h, + 1
                        qa[t][i2 + 2 * h] = (fq < nq && off < row_bytes) ? __ldg(reinterpret_cast<const uint32_t *>(src + off)) : 0u;
                    }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes of sQ -> tensor-core reads
        named_sync<1, kConsThreads>();
        // stage `st` of the ring has been read by this CTA's MMAs: one arrival on its `empty` barrier in every CTA of
        // the cluster (each producer multicasts into all of them)
        auto release = [&](uint32_t st) {
            if (csize == 1) {
                if (et == 0) mbar_arrive(&empty[st]);
            } else if (et < (int)csize) {
                mbar_arrive_remote(mapa_u32(smem_u32(&empty[st]), (uint32_t)et));
            }
        };
        // ===== epilogue: this thread's query against 128 rows per tile =====
        uint32_t thr = 0xFFFFFFFFu, cnt = 0;
        // pre-test bound in the raw accumulator domain; -inf: everything passes until the first compaction
        float thr_dot = -__int_as_float(0x7f800000);
        float nq_norm = 1.0f;
        if constexpr (kOp == 2) nq_norm = live ? *reinterpret_cast<const float *>(q16 + (size_t)q * q16_pitch + dim) : 1.0f;
        if constexpr (kOp == 3) nq_norm = live ? q_norm2[q] : 0.0f; // |q|^2
        // kOp 4: the exact int32 |q|^2, and the pre-test bound on the int32 distance e: a row can only pass the key test
        // (float)e < T if e < T, and every stored T is an integer (a rounded integer), so e < thr_e = T is exact.
        // INT_MIN: slots without a query never pass (e >= 0)
        const int *irn2 = reinterpret_cast<const int *>(row_norm2);
        int nq_int = 0, thr_e = live ? INT_MAX : INT_MIN;
        if constexpr (kOp == 4) nq_int = live ? reinterpret_cast<const int *>(q_norm2)[q] : 0;
        float smax[kSample ? kSliceSets : 1][kQN / 32]; // kSample: running maxima of the pre-test value per slice (largest = smallest distance)
#pragma unroll
        for (int x = 0; x < (kSample ? kSliceSets : 1); x++)
#pragma unroll
            for (int h = 0; h < kQN / 32; h++) smax[x][h] = -__int_as_float(0x7f800000);
        if (!live) thr_dot = __int_as_float(0x7f800000); // slots without a query: nothing ever passes
        // kFixed: the bound is tested on the accumulator fragment itself, where this thread holds queries
        // fq[i2] = 16 ew + lane / 4 + 8 i2 (i2 = 0, 1) against 32 rows of each tile
        uint32_t fthr[2];
        float fthr_dot[2], fnq[2];
        // 8-bit fixed radius: the radius, the integer bound of the inner-product / L2 pre-test, |q|^2 (L2)
        float frad[2];
        int fix[2], fnqi[2];
        // kOp 5: the scales s_q of the two fragment queries (1 for slots without a query)
        float fsq[2] = {1.0f, 1.0f};
        float frq[2] = {1.0f, 1.0f}; // kFixed: fl(1 / s_q) (q8_dot_bound)
        if constexpr (kQ8) {
#pragma unroll
            for (int i2 = 0; i2 < 2; i2++) {
                const uint32_t fq = qw + 16 * ew + (lane >> 2) + 8 * i2;
                if (fq < nq) fsq[i2] = *reinterpret_cast<const float *>(q16 + (size_t)fq * q16_pitch + row_bytes);
                if constexpr (kFixed) frq[i2] = __frcp_rn(fsq[i2]);
            }
        }
        if constexpr (kFixed && kInt && !kQ8) {
#pragma unroll
            for (int i2 = 0; i2 < 2; i2++) {
                const uint32_t fq = qw + 16 * ew + (lane >> 2) + 8 * i2;
                const bool flive = fq < nq;
                frad[i2] = flive ? thr_fixed[fq] : __int_as_float(0x7fffffff); // slots without a query: a NaN radius keeps nothing
                fix[i2] = range_int_bound(frad[i2]);
                fnqi[i2] = (kOp == 4 && flive) ? reinterpret_cast<const int *>(q_norm2)[fq] : 0;
                // cosine: d = 1 - fl(D / fl(nr nq)) with D = fl(dot).  d <= r implies D >= nr nq (t - 1.3e-7 (1 + |r|)), t = 1 - r
                // (relative rounding 2^-24 of the subtraction, the division, D and the norm product, |D / P| <= 1 + 4 ulp by
                // Cauchy-Schwarz on rows that carry their own norm).  The pre-test D >= fl(nr fthr_dot) with fthr_dot =
                // fl(nq fl(t - 1e-6 (1 + |r|))) rounds three more times (< 2.4e-7 (1 + |r|) nr nq) and so never drops such a row.
                fnq[i2] = (kOp == 2 && flive) ? *reinterpret_cast<const float *>(q16 + (size_t)fq * q16_pitch + dim) : 0.0f;
                fthr_dot[i2] = fnq[i2] * ((1.0f - frad[i2]) - 1e-6f * (1.0f + fabsf(frad[i2])));
            }
        }
        if constexpr (kFixed && (!kInt || kQ8)) {
#pragma unroll
            for (int i2 = 0; i2 < 2; i2++) {
                const uint32_t fq = qw + 16 * ew + (lane >> 2) + 8 * i2;
                const bool flive = fq < nq;
                fnq[i2] = (kOp == 3 && flive) ? q_norm2[fq] : 0.0f; // |q|^2
                // fixed admission bound (a distance): keep every row with approximate distance < T
                const float T = flive ? thr_fixed[fq] : -__int_as_float(0x7f800000);
                fthr[i2] = orderable_key(T);
                if constexpr (kOpE == 0) { // d < T  <=>  dot > 1 - T; slack: the rounding of the two subtractions
                    const float t = 1.0f - T;
                    fthr_dot[i2] = t - (4e-7f + 2.4e-7f * fabsf(t));
                } else {
                    fthr_dot[i2] = 0.5f * (fnq[i2] - T) - 2e-6f * (fabsf(fnq[i2]) + fabsf(T));
                }
                if (!(T == T)) fthr_dot[i2] = -__int_as_float(0x7f800000), fthr[i2] = 0xFFFFFFFFu; // NaN bound: keep everything (-> overflow -> next tier)
                if (!flive) fthr_dot[i2] = __int_as_float(0x7f800000);
            }
        }
        uint32_t s = 0, ph = 0;
        const uint64_t bdesc_first = make_smem_desc(smem_u32(sB)), adesc_first = make_smem_desc(smem_u32(sQ + wq * 128));
        constexpr uint64_t kStageStep = kQStageBytes >> 4, kBlockStep = kQBlockBytes >> 4, kAKbStep = kQKbBytes >> 4;
        // kCons warpgroups take tiles i = cw, cw + kCons, ...; a warpgroup steps its ring position past the stages of
        // the tiles the others take.  MMA issue stays in ring order: a warpgroup waits on a stage's `full` barrier only
        // once every earlier stage has been waited on, so that barrier is never more than one phase ahead of the wait.
        // kWide: both warpgroups take every tile, each against its own 64 queries, and walk the ring independently: the
        // producer refills a stage once both have released it, so neither is ever more than one ring ahead of the other, and
        // one warpgroup's drain and bound test run under the other's MMAs.  (Issuing every stage in turn, warpgroup 0 first,
        // left each one waiting through the other's bound test: DESIGN.md §4.2.)
        const uint32_t stages_per_tile = num_kb / kQKbPerStage;
        auto skip = [&](uint32_t n) {
            for (s += n; s >= nstages; s -= nstages) ph ^= 1;
        };
        if (kCons > 1 && !kWide) skip(stages_per_tile * cw);
        const long long t_pass = ca.now();
        for (uint32_t i = kWide ? 0 : cw; i < my_tiles; i += kWide ? 1 : kCons) {
            const uint32_t tile = (bx + i * gx) * tile_stride;
            if (kCons > 1 && !kWide && i >= (uint32_t)kCons) skip(stages_per_tile * (kCons - 1));
            ca.count(kCaTiles);
            float nrm[kQN / 32]; // kOp 2 / 3: lane l holds the norm / squared norm of rows h*32 + l of the tile
            int inrm[kQN / 32];  // kOp 4: the same, int32
            if constexpr (kOp == 4) {
#pragma unroll
                for (int h = 0; h < kQN / 32; h++) {
                    const uint32_t r = tile * kQN + h * 32 + lane;
                    inrm[h] = r < n_rows ? __ldg(irn2 + r) : 0;
                }
            }
            if constexpr (kOp == 3 && !kFixed) {
#pragma unroll
                for (int h = 0; h < kQN / 32; h++) {
                    const uint32_t r = tile * kQN + h * 32 + lane;
                    nrm[h] = r < n_rows ? __ldg(row_norm2 + r) : 0.0f;
                }
            }
            if constexpr (kOp == 2) {
#pragma unroll
                for (int h = 0; h < kQN / 32; h++) {
                    const uint32_t r = tile * kQN + h * 32 + lane;
                    nrm[h] = r < n_rows ? __ldg(reinterpret_cast<const float *>(shadow + (size_t)r * row_pitch + dim)) : 1.0f;
                }
            }
            // kFixed: acc[4 j + 2 i2 + c] holds row rbase + 8 j + c of the tile; squared L2 loads the squared norms of
            // each row pair (j) at once
            const uint32_t rbase = tile * kQN + 2 * (lane & 3);
            // kOp 5, fixed bound: the tile's scale s_t, loaded before the MMAs so that the bound test after the drain does not
            // wait for it
            float q8_st = 0.0f;
            if constexpr (kFrag && kQ8) q8_st = __ldg(row_norm2 + tile);
            float2 rn[(kFixed && kOp == 3) ? kQN / 8 : 1];
            if constexpr (kFixed && kOp == 3) {
#pragma unroll
                for (int j = 0; j < kQN / 8; j++) {
                    const uint32_t r = rbase + 8 * j;
                    if (r + 1 < n_rows)
                        rn[j] = __ldg(reinterpret_cast<const float2 *>(row_norm2 + r));
                    else
                        rn[j] = make_float2(r < n_rows ? __ldg(row_norm2 + r) : 0.0f, 0.0f);
                }
            }
            if constexpr (kCons > 1 && !kWide) {
                static_assert(kCons == 2, "the hand-off pairs two warpgroups");
                // hand-off: the warpgroup of tile i - 1 has issued its last MMAs (warpgroup cw waits on barrier 2 + cw)
                const long long t_handoff = ca.now();
                if (i != 0) {
                    if (cw == 0)
                        named_sync<2, 2 * 128>();
                    else
                        named_sync<3, 2 * 128>();
                }
                ca.add(kCaHandoff, t_handoff);
            }
            // ===== D[64 queries x 128 rows] (+)= Q[smem] * rows[smem]^T, per warpgroup =====
            Acc acc[64];
            uint32_t prev = 0;
            // one ring stage (K blocks kb0, kb0 + 1): wait for it, issue(bd) its MMAs against the stage's B descriptor, hand
            // the tile on after its last stage, release the stage before
            auto stage = [&](uint32_t kb0, auto issue) {
                const long long t_wait = ca.now();
                mbar_wait_spin(&full[s], ph);
                const long long t_issue = ca.now();
                ca.add(kCaWait, t_wait);
                wg_fence(); // the accumulator registers are handed to the MMA pipe for this stage's run
                issue(bdesc_first + (uint64_t)s * kStageStep);
                wg_commit();
                if constexpr (kCons > 1 && !kWide) { // the tile's last MMAs are issued: the other warpgroup may start the next tile
                    if (kb0 + kQKbPerStage >= num_kb && i + 1 < my_tiles) {
                        if (cw == 0)
                            named_arrive<3, 2 * 128>();
                        else
                            named_arrive<2, 2 * 128>();
                    }
                }
                ca.add(kCaIssue, t_issue);
                const long long t_wait1 = ca.now();
                wg_wait<1>(); // the previous stage's MMAs have retired (nothing to wait for on the first): its slot may be refilled
                ca.add(kCaWait1, t_wait1);
                if (kb0 != 0) release(prev);
                prev = s;
                if (++s == nstages) s = 0, ph ^= 1;
            };
            // x = 4 j + kk: K block j of the stage, 32-byte step kk inside its swizzled rows
            if constexpr (kRegKb > 0) { // K blocks 0 .. kRegKb - 1: A from registers, unrolled so that the indices are static
#pragma unroll
                for (int rs = 0; rs < kRegKb / kQKbPerStage; rs++)
                    stage(rs * kQKbPerStage, [&](uint64_t bd) {
#pragma unroll
                        for (int x = 0; x < 4 * kQKbPerStage; x++)
                            wgmma_f16_n128_ra(acc, qa[4 * kQKbPerStage * rs + x], bd + (x >> 2) * kBlockStep + 2 * (x & 3), (rs | x) != 0);
                    });
            }
            for (uint32_t kb0 = kRegKb; kb0 < num_kb; kb0 += kQKbPerStage)
                stage(kb0, [&](uint64_t bd) {
                    const uint64_t ad = adesc_first + (uint64_t)(kb0 - kRegKb) * kAKbStep;
#pragma unroll
                    for (int x = 0; x < 4 * kQKbPerStage; x++)
                        wgmma_n128<kInt, kVar>(acc, ad + (x >> 2) * kAKbStep + 2 * (x & 3), bd + (x >> 2) * kBlockStep + 2 * (x & 3),
                                               (kb0 | (uint32_t)x) != 0);
                });
            const long long t_epilogue = ca.now();
            wg_wait<0>();
            release(prev);
            wg_fence_operands(acc);
            // accumulator fragment: acc[4j + 2 i2 + c] = (query 16 ew + lane / 4 + 8 i2, row 8 j + 2 (lane % 4) + c)
            if constexpr (kSample && kQ8) {
                // int8 sample pass: for each of its two queries, c and 32-row chunk h, the thread's 4 rows 8 j + 2 (lane % 4) + c
                // (j = 4 h .. 4 h + 3) of the tile belong to slice (lane % 4, c, h).  The largest accumulator of the four has
                // their smallest approximate distance 1 - fl(fl(s_q s_t) acc) (int -> float rounding and the product with
                // s_q s_t >= 0 are monotone), so only that one is converted; smax[h][2 i2 + c] keeps the largest such dot
                // product of the slice.  Rows past n_rows (zero or stale shadow bytes) never count.
                const bool tail = tile * kQN + kQN > n_rows;
#pragma unroll
                for (int i2 = 0; i2 < 2; i2++) {
                    const float sqt = __fmul_rn(fsq[i2], q8_st);
#pragma unroll
                    for (int c = 0; c < 2; c++)
#pragma unroll
                        for (int h = 0; h < kQN / 32; h++) {
                            int v[4];
#pragma unroll
                            for (int u = 0; u < 4; u++) {
                                const int j = 4 * h + u;
                                v[u] = (!tail || rbase + 8 * j + c < n_rows) ? (int)acc[4 * j + 2 * i2 + c] : INT_MIN;
                            }
                            const int mx = max(__vimax3_s32(v[0], v[1], v[2]), v[3]);
                            if (mx != INT_MIN) smax[h][2 * i2 + c] = fmaxf(smax[h][2 * i2 + c], __fmul_rn(sqt, __int2float_rn(mx)));
                        }
                }
                continue;
            }
            if constexpr (kFixed && kQ8) {
                // int8 shadow: the bound dot > fthr_dot becomes one integer bound per query on this tile's accumulators
                // (q8_dot_bound); the rare survivors take the float distance and the exact key comparison, as kOp 0
                const float st = q8_st, rst = __frcp_rn(st);
#pragma unroll
                for (int i2 = 0; i2 < 2; i2++) {
                    const float sqt = __fmul_rn(fsq[i2], st);
                    const int ti = q8_dot_bound(fthr_dot[i2], frq[i2], rst);
                    // the max of the query's 32 values: a tree of three-input maxima
                    int m3[11];
#pragma unroll
                    for (int g = 0; g < 10; g++)
                        m3[g] = __vimax3_s32((int)acc[4 * ((3 * g) >> 1) + 2 * i2 + ((3 * g) & 1)],
                                             (int)acc[4 * ((3 * g + 1) >> 1) + 2 * i2 + ((3 * g + 1) & 1)],
                                             (int)acc[4 * ((3 * g + 2) >> 1) + 2 * i2 + ((3 * g + 2) & 1)]);
                    m3[10] = max((int)acc[4 * 15 + 2 * i2], (int)acc[4 * 15 + 2 * i2 + 1]); // values 30, 31
                    const int mx = __vimax3_s32(__vimax3_s32(m3[0], m3[1], m3[2]), __vimax3_s32(m3[3], m3[4], m3[5]),
                                                __vimax3_s32(__vimax3_s32(m3[6], m3[7], m3[8]), m3[9], m3[10]));
                    uint32_t pass = 0; // bit 2 j + c: acc[4 j + 2 i2 + c]
                    if (mx > ti) {
#pragma unroll
                        for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                            for (int c = 0; c < 2; c++)
                                if ((int)acc[4 * j + 2 * i2 + c] > ti) pass |= 1u << (2 * j + c);
                    }
                    if (pass && tile * kQN + kQN > n_rows) { // rows past the end (zero or stale shadow bytes)
#pragma unroll
                        for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                            for (int c = 0; c < 2; c++)
                                if (rbase + 8 * j + c >= n_rows) pass &= ~(1u << (2 * j + c));
                    }
                    while (pass) {
                        const int b = __ffs(pass) - 1;
                        pass &= pass - 1;
                        uint32_t raw = 0;
#pragma unroll
                        for (int x = 0; x < 32; x++)
                            if (x == b) raw = acc[4 * (x >> 1) + 2 * i2 + (x & 1)];
                        const uint32_t row = rbase + 8 * (b >> 1) + (b & 1);
                        const uint32_t key = orderable_key(__fsub_rn(1.0f, __fmul_rn(sqt, __int2float_rn((int)raw))));
                        if (key < fthr[i2]) {
                            const int qs = wq + 16 * ew + (lane >> 2) + 8 * i2;
                            const uint32_t slot = atomicAdd(&qcount[qs], 1u);
                            if (slot < (uint32_t)kQListCap) lists[slot * kQListStride + qs] = ((uint64_t)key << 32) | row;
                        }
                    }
                }
                ca.add(kCaEpilogue, t_epilogue);
                continue;
            }
            if constexpr (kFixed && kInt) {
                // 8-bit fixed radius: a conservative pre-test on the integer dot products (exact for inner product and L2,
                // range_int_bound), then the epilogue's own float distance and the range test d <= r on the rare survivors.
                // Every entry of a list is a hit with its final distance; a list that runs full sets the overflow flag.
                uint32_t pass2[2] = {0u, 0u}; // bit 2 j + c: acc[4 j + 2 i2 + c]
                if constexpr (kOp == 1) { // 1 - dot <= X  <=>  dot >= 1 - X: one compare against the largest dot decides most rows
#pragma unroll
                    for (int i2 = 0; i2 < 2; i2++) {
                        int mx = (int)acc[2 * i2];
#pragma unroll
                        for (int x = 1; x < 32; x++) mx = max(mx, (int)acc[4 * (x >> 1) + 2 * i2 + (x & 1)]);
                        if (1 - mx <= fix[i2]) {
#pragma unroll
                            for (int x = 0; x < 32; x++)
                                if (1 - (int)acc[4 * (x >> 1) + 2 * i2 + (x & 1)] <= fix[i2]) pass2[i2] |= 1u << x;
                        }
                    }
                } else { // per row: |row|^2 (L2) or the row norm (cosine) from the lane that loaded it
#pragma unroll
                    for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const int src = 8 * (j & 3) + 2 * (lane & 3) + c; // row 8 j + 2 (lane % 4) + c of the tile
                            if constexpr (kOp == 4) {
                                const int rn = __shfl_sync(0xFFFFFFFFu, inrm[j >> 2], src);
#pragma unroll
                                for (int i2 = 0; i2 < 2; i2++)
                                    if (rn + fnqi[i2] - 2 * (int)acc[4 * j + 2 * i2 + c] <= fix[i2]) pass2[i2] |= 1u << (2 * j + c);
                            } else {
                                const float nr = __shfl_sync(0xFFFFFFFFu, nrm[j >> 2], src);
#pragma unroll
                                for (int i2 = 0; i2 < 2; i2++)
                                    if (__int2float_rn((int)acc[4 * j + 2 * i2 + c]) >= nr * fthr_dot[i2]) pass2[i2] |= 1u << (2 * j + c);
                            }
                        }
                }
#pragma unroll
                for (int i2 = 0; i2 < 2; i2++) {
                    uint32_t pass = pass2[i2];
                    if (pass && tile * kQN + kQN > n_rows) { // rows past the end (TMA zero fill)
#pragma unroll
                        for (int x = 0; x < 32; x++)
                            if (rbase + 8 * (x >> 1) + (x & 1) >= n_rows) pass &= ~(1u << x);
                    }
                    while (pass) {
                        const int b = __ffs(pass) - 1;
                        pass &= pass - 1;
                        uint32_t raw = 0;
#pragma unroll
                        for (int x = 0; x < 32; x++)
                            if (x == b) raw = acc[4 * (x >> 1) + 2 * i2 + (x & 1)];
                        const uint32_t row = rbase + 8 * (b >> 1) + (b & 1);
                        float d; // the expressions of the adaptive-list epilogue below
                        if constexpr (kOp == 1) {
                            d = (float)(1 - (int)raw);
                        } else if constexpr (kOp == 2) {
                            const float nr = __ldg(reinterpret_cast<const float *>(shadow + (size_t)row * row_pitch + dim));
                            d = __fsub_rn(1.0f, __fdiv_rn((float)(int)raw, __fmul_rn(nr, fnq[i2])));
                        } else {
                            d = __int2float_rn(__ldg(irn2 + row) + fnqi[i2] - 2 * (int)raw);
                        }
                        bool hit = d <= frad[i2]; // the reference's inclusive range test: NaN never passes, -0 == +0
                        if constexpr (kFilt) { // a hit counts only if the query's filter holds the row
                            if (hit) hit = (__ldg(filt_row(q_base + 16 * ew + (lane >> 2) + 8 * i2) + (row >> 5)) >> (row & 31)) & 1u;
                        }
                        if (hit) {
                            const int qs = wq + 16 * ew + (lane >> 2) + 8 * i2;
                            const uint32_t slot = atomicAdd(&qcount[qs], 1u);
                            if (slot < (uint32_t)kQListCap) lists[slot * kQListStride + qs] = ((uint64_t)orderable_key(d) << 32) | row;
                        }
                    }
                }
                ca.add(kCaEpilogue, t_epilogue);
                continue;
            }
            if constexpr (kFixed && !kInt) {
                // With a fixed bound only ~k * (rows / sample rows) rows of the whole corpus pass: for each of its two
                // queries the thread takes the max of its 32 values and ONE compare decides the common case.  The rare
                // survivors take the exact distance and key comparison and append to the query's list, unordered, at a
                // slot from the query's shared counter; a count past the capacity is an overflow.
#pragma unroll
                for (int i2 = 0; i2 < 2; i2++) {
                    uint32_t pass = 0; // bit 2 j + c: acc[4 j + 2 i2 + c]
                    if constexpr (kOp == 0) {
                        float m8[8];
#pragma unroll
                        for (int g = 0; g < 8; g++)
                            m8[g] = fmaxf(fmaxf(acc[8 * g + 2 * i2], acc[8 * g + 2 * i2 + 1]), fmaxf(acc[8 * g + 4 + 2 * i2], acc[8 * g + 5 + 2 * i2]));
                        const float mx = fmaxf(fmaxf(fmaxf(m8[0], m8[1]), fmaxf(m8[2], m8[3])), fmaxf(fmaxf(m8[4], m8[5]), fmaxf(m8[6], m8[7])));
                        if (mx > fthr_dot[i2]) {
#pragma unroll
                            for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                                for (int c = 0; c < 2; c++)
                                    if (acc[4 * j + 2 * i2 + c] > fthr_dot[i2]) pass |= 1u << (2 * j + c);
                        }
                    } else { // d < d_thr  <=>  dot > |row|^2 / 2 + (|q|^2 - d_thr) / 2, loosened for the rounding of both sides
#pragma unroll
                        for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                            for (int c = 0; c < 2; c++)
                                if (acc[4 * j + 2 * i2 + c] > fmaf(c ? rn[j].y : rn[j].x, 0.499999f, fthr_dot[i2])) pass |= 1u << (2 * j + c);
                    }
                    if (pass && tile * kQN + kQN > n_rows) { // rows past the end (TMA zero fill / stale shadow bytes)
#pragma unroll
                        for (int j = 0; j < kQN / 8; j++)
#pragma unroll
                            for (int c = 0; c < 2; c++)
                                if (rbase + 8 * j + c >= n_rows) pass &= ~(1u << (2 * j + c));
                    }
                    while (pass) {
                        const int b = __ffs(pass) - 1;
                        pass &= pass - 1;
                        float raw = 0.0f;
#pragma unroll
                        for (int x = 0; x < 32; x++)
                            if (x == b) raw = acc[4 * (x >> 1) + 2 * i2 + (x & 1)];
                        const uint32_t row = rbase + 8 * (b >> 1) + (b & 1);
                        float d;
                        if constexpr (kOp == 0)
                            d = 1.0f - raw;
                        else
                            d = __fsub_rn(__fadd_rn(fnq[i2], __ldg(row_norm2 + row)), __fmul_rn(2.0f, raw));
                        const uint32_t key = orderable_key(d);
                        bool admit = key < fthr[i2];
                        if constexpr (kFilt) { // a row below the bound enters the list only if the query's filter holds it
                            if (admit) admit = (__ldg(filt_row(q_base + 16 * ew + (lane >> 2) + 8 * i2) + (row >> 5)) >> (row & 31)) & 1u;
                        }
                        if (admit) {
                            const int qs = wq + 16 * ew + (lane >> 2) + 8 * i2;
                            const uint32_t slot = atomicAdd(&qcount[qs], 1u);
                            if (slot < (uint32_t)kQListCap) lists[slot * kQListStride + qs] = ((uint64_t)key << 32) | row;
                        }
                    }
                }
                ca.add(kCaEpilogue, t_epilogue);
                continue;
            }
            asm volatile("bar.sync 1, 128;" ::: "memory"); // the previous tile's reads of sacc are done
            float tsqt[2] = {0.0f, 0.0f}; // kOp 5: fl(s_q s_t) of the fragment's two queries on this tile
            if constexpr (kQ8) {
                const float st = __ldg(row_norm2 + tile);
                tsqt[0] = __fmul_rn(fsq[0], st), tsqt[1] = __fmul_rn(fsq[1], st);
            }
#pragma unroll
            for (int j = 0; j < kQN / 8; j++) {
                const int m = 16 * ew + (lane >> 2), n = 8 * j + 2 * (lane & 3);
                uint32_t b[4];
#pragma unroll
                for (int x = 0; x < 4; x++) {
                    if constexpr (kQ8)
                        b[x] = __float_as_uint(__fmul_rn(tsqt[x >> 1], __int2float_rn((int)acc[4 * j + x])));
                    else if constexpr (kInt)
                        b[x] = acc[4 * j + x];
                    else
                        b[x] = __float_as_uint(acc[4 * j + x]);
                }
                *reinterpret_cast<uint2 *>(sacc + m * kQAccStride + n) = make_uint2(b[0], b[1]);
                *reinterpret_cast<uint2 *>(sacc + (m + 8) * kQAccStride + n) = make_uint2(b[2], b[3]);
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            uint32_t v[kQN / 32][32];
            {
                const uint32_t *mine = sacc + (et & (kQM - 1)) * kQAccStride; // slots >= kQM read a copy they never use
#pragma unroll
                for (int h = 0; h < kQN / 32; h++)
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const uint4 w = *reinterpret_cast<const uint4 *>(mine + h * 32 + 4 * u);
                        v[h][4 * u] = w.x, v[h][4 * u + 1] = w.y, v[h][4 * u + 2] = w.z, v[h][4 * u + 3] = w.w;
                    }
            }
#pragma unroll
            for (int h = 0; h < kQN / 32; h++) {
                const uint32_t row0 = tile * kQN + h * 32;
                // kFilt: the filter's word for the 32 rows of this chunk (no bit is set past the last row)
                uint32_t fw = 0xFFFFFFFFu;
                if constexpr (kFilt) fw = (live && row0 < n_rows) ? __ldg(filt_row(q) + (row0 >> 5)) : 0u;
                if constexpr (kSample) {
                    // largest dot (cosine / inner product) or largest dot - |row|^2 / 2 (squared L2) of the chunk
                    float mx = -__int_as_float(0x7f800000);
                    const bool tail = row0 + 32 > n_rows; // rows past the end (zero fill / stale shadow bytes) must not count
                    if constexpr (kFilt) { // the maximum over the chunk's filtered rows only
#pragma unroll
                        for (int j = 0; j < 32; j++) {
                            float u = __uint_as_float(v[h][j]);
                            if constexpr (kOpE != 0) u = fmaf(__shfl_sync(0xFFFFFFFFu, nrm[h], j), -0.5f, u);
                            if ((fw >> j) & 1u) mx = fmaxf(mx, u);
                        }
                    } else if constexpr (kOpE == 0) {
                        if (!tail) {
                            float m8[8];
#pragma unroll
                            for (int g = 0; g < 8; g++)
                                m8[g] = fmaxf(fmaxf(__uint_as_float(v[h][4 * g]), __uint_as_float(v[h][4 * g + 1])),
                                              fmaxf(__uint_as_float(v[h][4 * g + 2]), __uint_as_float(v[h][4 * g + 3])));
                            mx = fmaxf(fmaxf(fmaxf(m8[0], m8[1]), fmaxf(m8[2], m8[3])), fmaxf(fmaxf(m8[4], m8[5]), fmaxf(m8[6], m8[7])));
                        } else {
#pragma unroll
                            for (int j = 0; j < 32; j++)
                                if (row0 + j < n_rows) mx = fmaxf(mx, __uint_as_float(v[h][j]));
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; j++) {
                            const float u = fmaf(__shfl_sync(0xFFFFFFFFu, nrm[h], j), -0.5f, __uint_as_float(v[h][j]));
                            if (!tail || row0 + j < n_rows) mx = fmaxf(mx, u);
                        }
                    }
                    // slice set = tile counter mod kSliceSets: a uniform switch keeps the register indices static
#pragma unroll
                    for (int x = 0; x < kSliceSets; x++)
                        if ((int)(i % (uint32_t)kSliceSets) == x) smax[kSample ? x : 0][h] = fmaxf(smax[kSample ? x : 0][h], mx);
                    continue;
                }
                // pre-test on the raw dot product against a slightly loose bound (a few instructions per value);
                // the few survivors take the exact distance and key comparison below
                uint32_t pass = 0;
#pragma unroll
                for (int j = 0; j < 32; j++) {
                    bool p;
                    if constexpr (kOpE == 0)
                        p = __uint_as_float(v[h][j]) > thr_dot;
                    else if constexpr (kOp == 1)
                        p = (float)(int)v[h][j] > thr_dot;
                    else if constexpr (kOp == 2)
                        p = (float)(int)v[h][j] > __shfl_sync(0xFFFFFFFFu, nrm[h], j) * thr_dot - 0.01f;
                    else if constexpr (kOp == 4)
                        p = __shfl_sync(0xFFFFFFFFu, inrm[h], j) + nq_int - 2 * (int)v[h][j] < thr_e;
                    else // d < d_thr  <=>  dot > |row|^2 / 2 + (|q|^2 - d_thr) / 2, loosened for the rounding of both sides
                        p = __uint_as_float(v[h][j]) > fmaf(__shfl_sync(0xFFFFFFFFu, nrm[h], j), 0.499999f, thr_dot);
                    if (p) pass |= 1u << j;
                }
                if (row0 + 32 > n_rows) pass &= (n_rows > row0) ? ((1u << (n_rows - row0)) - 1u) : 0u; // TMA zero fill past the end
                if constexpr (kFilt) pass &= fw;
                while (pass) {
                    const int j = __ffs(pass) - 1;
                    pass &= pass - 1;
                    uint32_t raw = 0;
#pragma unroll
                    for (int x = 0; x < 32; x++)
                        if (x == j) raw = v[h][x];
                    float d;
                    if constexpr (kOpE == 0)
                        d = 1.0f - __uint_as_float(raw);
                    else if constexpr (kOp == 1)
                        d = (float)(1 - (int)raw);
                    else if constexpr (kOp == 2) {
                        const uint32_t r = row0 + j; // rare path: re-read the norm (L1/L2 hit) instead of a divergent shuffle
                        const float nr = __ldg(reinterpret_cast<const float *>(shadow + (size_t)r * row_pitch + dim));
                        d = __fsub_rn(1.0f, __fdiv_rn((float)(int)raw, __fmul_rn(nr, nq_norm)));
                    } else if constexpr (kOp == 4) {
                        d = __int2float_rn(__ldg(irn2 + row0 + j) + nq_int - 2 * (int)raw); // rare path: re-read, as kOp 2
                    } else {
                        d = __fsub_rn(__fadd_rn(nq_norm, __ldg(row_norm2 + row0 + j)), __fmul_rn(2.0f, __uint_as_float(raw)));
                    }
                    const uint32_t key = orderable_key(d);
                    if (key < thr) {
                        lists[cnt * kQListStride + et] = ((uint64_t)key << 32) | (row0 + j);
                        cnt++;
                    }
                }
                // lists that ran past the trigger are cut back to the best `keep` by the whole warp
                uint32_t m = __ballot_sync(0xFFFFFFFFu, cnt > kQTrigger);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const uint32_t c = __shfl_sync(0xFFFFFFFFu, cnt, src);
                    const uint32_t worst = select_keep<kEpl>(lists, ew * 32 + src, c, keep, lane);
                    if (lane == src) {
                        cnt = keep;
                        thr = worst;
                        // d < d_thr needs dot > t = 1 - d_thr (times the norms for the integer cosine); the slack covers
                        // the rounding of the subtractions, of int -> float and of the norm product
                        const float t = 1.0f - key_to_float(thr);
                        if constexpr (kOpE == 0)
                            thr_dot = t - 4e-7f;
                        else if constexpr (kOp == 1)
                            thr_dot = t - (fabsf(t) * 1e-6f + 2.0f);
                        else if constexpr (kOp == 2) {
                            const float tq = t * nq_norm;
                            thr_dot = tq - fabsf(tq) * 4e-6f;
                        } else if constexpr (kOp == 4) {
                            thr_e = __float2int_ru(key_to_float(thr)); // a finite distance in [0, 2^28]
                        } else {
                            const float dthr = key_to_float(thr);
                            thr_dot = 0.5f * (nq_norm - dthr) - 2e-6f * (fabsf(nq_norm) + fabsf(dthr));
                        }
                    }
                }
            }
        }
        ca.add(kCaPass, t_pass);
        if (kFixed && et == 0) ca.flush(cta, cw);
        // publish: cand_out[q][blockIdx.x][keep], kEmptySlot padded
        __syncwarp();
        if constexpr (kFixed) {
            // every append of the CTA is done; consumer warp pw publishes query slots per * pw .. per * pw + per - 1.
            // keep == kQListCap here (plan_coarse), so a list that did not overflow is published whole.  More rows below
            // the bound than the list holds: overflow, the query goes to the next tier.
            named_sync<1, kConsThreads>();
            constexpr int per = kCtaQ / (4 * kCons);
            const int pw = 4 * cw + ew;
            for (int qs = per * pw; qs < per * pw + per; qs++) {
                const uint32_t qq = q_base + qs;
                if (qq >= nq) break;
                const uint32_t n = qcount[qs], c = min(n, (uint32_t)kQListCap);
                uint64_t *dst = cand_out + ((size_t)qq * gx + bx) * keep;
                if constexpr (kQ8) { // the list's entries only: its reader takes their number from list_count
                    for (uint32_t r = lane; r < c; r += 32) dst[r] = lists[r * kQListStride + qs];
                } else {
                    for (uint32_t r = lane; r < keep; r += 32) dst[r] = r < c ? lists[r * kQListStride + qs] : kEmptySlot;
                }
                if (lane == 0 && list_count) list_count[(size_t)qq * gx + bx] = c;
                if (lane == 0 && n > (uint32_t)kQListCap) overflow[qq] = 1u;
            }
        }
        if constexpr (kSample && kFrag) {
            // the slice minima of the fragment's two queries: slice (lane % 4, c, h) at composite 8 (lane % 4) + 4 c + h
#pragma unroll
            for (int i2 = 0; i2 < 2; i2++) {
                const uint32_t fq = qw + 16 * ew + (lane >> 2) + 8 * i2;
                if (fq >= nq) continue;
                uint64_t *dst = cand_out + ((size_t)fq * gx + bx) * keep + 8 * (lane & 3);
#pragma unroll
                for (int c = 0; c < 2; c++)
#pragma unroll
                    for (int h = 0; h < kQN / 32; h++) {
                        const float m = smax[h][2 * i2 + c];
                        dst[4 * c + h] = m > -__int_as_float(0x7f800000) ? (uint64_t)orderable_key(1.0f - m) << 32 : kEmptySlot;
                    }
            }
        }
        if constexpr (kSample && !kFrag) { // keep == 32: the slice minima as composites (the row id is not needed by threshold_kernel)
            if (live) {
                uint64_t *dst = cand_out + ((size_t)q * gx + bx) * keep;
#pragma unroll
                for (int x = 0; x < kSliceSets; x++)
#pragma unroll
                    for (int h = 0; h < kQN / 32; h++) {
                        const float m = smax[kSample ? x : 0][h];
                        uint64_t c = kEmptySlot;
                        if (m > -__int_as_float(0x7f800000)) {
                            const float d = kOpE == 0 ? 1.0f - m : __fsub_rn(nq_norm, __fmul_rn(2.0f, m));
                            c = (uint64_t)orderable_key(d) << 32;
                        }
                        if ((uint32_t)(x * (kQN / 32) + h) < keep) dst[x * (kQN / 32) + h] = c;
                    }
            }
        }
        for (int src = 0; src < ((kSample || kFixed) ? 0 : 32); src++) {
            uint32_t c = __shfl_sync(0xFFFFFFFFu, cnt, src);
            const uint32_t qq = q_base + ew * 32 + src;
            if (c > keep) {
                select_keep<kEpl>(lists, ew * 32 + src, c, keep, lane);
                c = keep;
            }
            if (ew * 32 + src < kQM && qq < nq) {
                // unordered: final_select (direct routes) and refine_kernel (fp32 route) take the lists in any order
                uint64_t *dst = cand_out + ((size_t)qq * gx + bx) * keep;
                __syncwarp();
                for (uint32_t r = lane; r < keep; r += 32) dst[r] = r < c ? lists[r * kQListStride + ew * 32 + src] : kEmptySlot;
            }
        }
    }
    __syncthreads();
    if (csize > 1) cluster_sync_all(); // no CTA may exit while peers can still write its shared memory / barriers
}

// fp32 rows -> fp16 (round to nearest even) shadow rows; 8 elements per thread, dim % 8 == 0
__global__ void __launch_bounds__(256) to_f16_kernel(const uint8_t *__restrict__ src, size_t spitch, uint32_t dim, uint32_t first,
                                                     uint32_t n, uint8_t *__restrict__ dst, size_t dpitch) {
    const uint32_t per_row = dim / 8;
    const size_t total = (size_t)n * per_row;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t r = first + (uint32_t)(i / per_row), c = (uint32_t)(i % per_row);
        const float4 *p = reinterpret_cast<const float4 *>(src + (size_t)r * spitch) + 2 * c;
        const float4 x = p[0], y = p[1];
        __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
        __half2 h2 = __floats2half2_rn(y.x, y.y), h3 = __floats2half2_rn(y.z, y.w);
        uint4 o;
        o.x = *reinterpret_cast<uint32_t *>(&h0);
        o.y = *reinterpret_cast<uint32_t *>(&h1);
        o.z = *reinterpret_cast<uint32_t *>(&h2);
        o.w = *reinterpret_cast<uint32_t *>(&h3);
        reinterpret_cast<uint4 *>(dst + (size_t)r * dpitch)[c] = o;
    }
}

// ------------------------------------------------------------------------------------------------
// stages 2 + 3 in one kernel, one CTA per query: exact rescoring of the candidates that can still matter, the exact
// top-k, and the completeness proof.
//
//   * a_k = the k-th smallest APPROXIMATE distance over all candidate lists of the query (radix select on the keys).
//     With |approx - exact| <= eps, the k best-approx candidates all have exact <= a_k + eps, so the k-th exact distance
//     e_k <= a_k + eps; a candidate with approx > a_k + 2 eps has exact > a_k + eps >= e_k and cannot be among the k
//     best: only candidates with approx <= a_k + 2 eps are re-read from the fp32 corpus (a few dozen rows instead of
//     lists x keep = 1,776) and scored with the bit-exact arithmetic of distance_core.cuh.
//   * proof (as before): a row that is NOT among the candidates of its list has approx >= the list's worst kept
//     approx a_w, hence exact >= a_w - eps.  If a_w - eps > e_k for every FULL list, nothing was missed.
//   eps: unit vectors (cosine): the constant `eps`.  Otherwise (q_norm2 != NULL) it scales with the norms — fp16 RN
//   operands give |dot error| <= eps |a| |q| (Cauchy-Schwarz; `eps` already holds the accumulation slack)
//   + 2^-24 sqrt(D) (|a| + |q|) for elements below the fp16 normal range; |a| <= max_norm for every row.  L2: twice
//   that (the -2 dot term) + the fp32 rounding of the squared norms, (D + 4) 2^-23 (max_norm^2 + |q|^2).
//   q_index (nullable): second tier — CTA i works on query q_index[i] of the original batch (its lists are stored at
//   position i); nq_dev (nullable) = number of live CTAs.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kRefineMaxSurv = 2048;     // survivors rescored per query, k <= kCoarseMaxK
constexpr uint32_t kRefineMaxSurvWide = 4096; // the same for k > kCoarseMaxK (32 KB)
constexpr uint32_t kRefineMaxLists = 256;     // lists per query of a counted first tier (one per thread of the scan)
// threads of refine_kernel: 16 warps share a query's survivors, each rescoring one row at a time, so that more rows are in
// flight per SM (a row is a few dependent rounds of loads from a random place in the corpus)
constexpr uint32_t kRefineThreads = 512;
// candidates refine_kernel packs into shared memory: lists with kEmptySlot padding (the fp16 shadow's 96-entry lists), lists of
// k > kCoarseMaxK, counted lists (the int8 shadow, DESIGN.md §4.2).  64 KB of packed candidates and the 19.5 KB of static
// shared memory leave two CTAs per SM: a batch of 256 queries stays resident in one wave on 132 SMs
constexpr uint32_t kRefineCapPadded = 2560, kRefineCapWide = 8192, kRefineCapCounted = 8192;

// |approx - exact| bound of one query (see above); q_norm2 == NULL: unit vectors.  q_eps (the int8 shadow): the bound of each
// query, computed with its quantization (quantize_queries_kernel)
__device__ __forceinline__ float query_eps(float eps, const float *q_norm2, uint32_t pos, float max_norm, uint32_t dim, bool l2,
                                           const float *q_eps = nullptr) {
    if (q_eps) return q_eps[pos];
    if (!q_norm2) return eps;
    const float qn2 = q_norm2[pos], qn = sqrtf(qn2);
    float e = eps * max_norm * qn + 5.97e-8f * sqrtf((float)dim) * (max_norm + qn);
    if (l2) e = 2.0f * e + (float)(dim + 4) * 1.2e-7f * (max_norm * max_norm + qn2);
    return e * 1.0001f;
}
// inclusive prefix sum of v over the threads of the block (warp scans, then the warp totals in wsum[blockDim.x / 32], at most
// 16); *total = the sum over the block.  Every thread must call it; wsum may be reused after the caller's next __syncthreads()
__device__ __forceinline__ uint32_t block_incl_scan(uint32_t v, uint32_t *wsum, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, v, o);
        if (lane >= o) v += y;
    }
    if (lane == 31) wsum[warp] = v;
    __syncthreads();
    uint32_t base = 0, all = 0;
    for (int w = 0; w < nw; w++) {
        const uint32_t x = wsum[w];
        if (w < warp) base += x;
        all += x;
    }
    *total = all;
    return v + base;
}

// k-th smallest key (high word) among the non-empty composites at(0), ..., at(total - 1) — block-wide radix select, 8 bits per
// pass; 0xFFFFFFFF when there are fewer than k.  256 to 512 threads; hist[256 + 16] and ctl[4] in shared memory.  The bin of the
// k-th key in each pass comes from a block-wide scan of the histogram: bin b is the one whose exclusive prefix is below the
// rank still sought and whose inclusive prefix reaches it (the last bin when none does), as a walk over the bins in order
// would find it.
template <class At>
__device__ __forceinline__ uint32_t block_kth_key(At at, uint32_t total, uint32_t k, uint32_t *hist, uint32_t *ctl) {
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) ctl[0] = 0, ctl[1] = k, ctl[2] = 0;
    __syncthreads();
    uint32_t cnt = 0;
    for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) cnt += at(i) != kEmptySlot;
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    if (lane == 0 && cnt) atomicAdd(&ctl[2], cnt);
    __syncthreads();
    if (ctl[2] < k) return 0xFFFFFFFFu;
    for (int shift = 24; shift >= 0; shift -= 8) {
        if (threadIdx.x < 256) hist[threadIdx.x] = 0;
        __syncthreads();
        const uint32_t prefix = ctl[0], rem = ctl[1];
        const uint32_t hi_mask = shift == 24 ? 0u : ~((1u << (shift + 8)) - 1u);
        for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
            const uint64_t c = at(i);
            if (c == kEmptySlot) continue;
            const uint32_t key = (uint32_t)(c >> 32);
            if (((key ^ prefix) & hi_mask) == 0) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        const uint32_t h = threadIdx.x < 256 ? hist[threadIdx.x] : 0u; // threads past the bins never hold the k-th
        uint32_t all;
        const uint32_t incl = block_incl_scan(h, hist + 256, &all), excl = incl - h;
        if (excl < rem && (incl >= rem || threadIdx.x == 255)) {
            ctl[0] = prefix | (threadIdx.x << shift);
            ctl[1] = rem - excl;
        }
        __syncthreads();
    }
    return ctl[0];
}

// Admission bound of the main pass from the SAMPLE pass (every tile_stride-th row tile): T[q] = (k-th smallest approximate
// distance among the sample's candidates) + 2 eps.  The k-th exact distance over the whole corpus e_k is at most the
// sample's, which is <= a_k + eps, so T - eps > e_k: a row the main pass drops (approx >= T) has exact >= T - eps > e_k.
// Also clears the overflow flags.  One CTA per query.
__global__ void __launch_bounds__(256) threshold_kernel(const uint64_t *__restrict__ cand, uint32_t nq, uint32_t lists_per_query,
                                                        uint32_t keep, uint32_t k, float eps, const float *__restrict__ q_norm2,
                                                        float max_norm, uint32_t dim, int l2, float *__restrict__ thr_out,
                                                        uint32_t *__restrict__ overflow, const float *__restrict__ q_eps) {
    __shared__ uint32_t hist[256 + 16];
    __shared__ uint32_t ctl[4];
    const uint32_t q = blockIdx.x;
    if (q >= nq) return;
    const uint64_t *mine = cand + (size_t)q * lists_per_query * keep;
    const uint32_t ak = block_kth_key([&](uint32_t i) { return mine[i]; }, lists_per_query * keep, k, hist, ctl);
    if (threadIdx.x == 0) {
        const float e = query_eps(eps, q_norm2, q, max_norm, dim, l2 != 0, q_eps);
        float T;
        if (ak == 0xFFFFFFFFu)
            T = __int_as_float(0x7f800000);
        else if (e == 0.0f) // 16-bit corpora: the GEMM result IS the distance — keep d <= a_k (the main pass tests d < T)
            T = key_to_float(ak + 1u);
        else
            T = key_to_float(ak) + (2.0f * e) * 1.001f + 1e-30f;
        thr_out[q] = T;
        overflow[q] = 0;
    }
}

// thr_T == NULL: adaptive lists (a full list's worst kept approximate distance bounds what its row range dropped).
// thr_T != NULL: lists of the fixed-bound pass — every list holds ALL rows of its range with approx < thr_T[pos] unless
//                overflow[pos] is set; what was dropped has approx >= thr_T[pos].
// kLab (hybrid batches, DESIGN.md §4.10): the exact composites carry the row's label row_label[row] instead of the row, so the
//      answer is the k smallest (distance, docId) — the order of the ragged gather over an ascending filter
template <int MT, uint32_t kSurv, bool kLab = false>
__global__ void __launch_bounds__(kRefineThreads) refine_kernel(const uint8_t *rows, size_t pitch, uint32_t dim, const uint8_t *queries,
                                                     size_t qpitch, uint32_t nq, uint32_t lists_per_query, uint32_t keep, uint32_t k,
                                                     const uint64_t *__restrict__ cand, float eps, const float *__restrict__ q_norm2,
                                                     float max_norm, uint32_t *__restrict__ ok, uint32_t ok_value, uint64_t *__restrict__ out,
                                                     const uint32_t *__restrict__ q_index, const uint32_t *__restrict__ nq_dev,
                                                     const float *__restrict__ thr_T, const uint32_t *__restrict__ overflow,
                                                     uint32_t smem_cap, const uint64_t *__restrict__ row_label, const float *__restrict__ q_eps,
                                                     const uint32_t *__restrict__ list_count) {
    using Tile = DistTile<DT_F32, MT, 1, 1>;
    __shared__ uint64_t surv[kSurv];
    __shared__ uint32_t hist[256 + 16];
    __shared__ uint32_t ctl[4];
    __shared__ uint32_t s_nsurv, s_bad, s_ncomp;
    __shared__ uint32_t s_off[kRefineMaxLists], s_cnt[kRefineMaxLists]; // list_count: offset and entries of each list
    if (nq_dev) nq = min(nq, *nq_dev);
    if (blockIdx.x >= nq) return;
    const uint32_t q = q_index ? q_index[blockIdx.x] : blockIdx.x; // query of the original batch
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr uint32_t kWarps = kRefineThreads / 32;
    const uint64_t *mine = cand + (size_t)blockIdx.x * lists_per_query * keep;
    uint32_t total = lists_per_query * keep;
    eps = query_eps(eps, q_norm2, blockIdx.x, max_norm, dim, MT == MT_L2, q_eps);
    if (threadIdx.x == 0) s_nsurv = 0, s_bad = 0, s_ncomp = 0;
    __syncthreads();
    // the lists are mostly empty slots (fixed-bound pass: ~15 of 96 per list): pack the real candidates into shared memory
    // once, so that the selection passes below do not re-read 57 KB of global memory five times per query
    extern __shared__ uint64_t s_cand[];
    if (list_count) {
        // counted lists (the int8 shadow's fixed pass): list l holds s_cnt[l] entries from its slot 0 and nothing after them.
        // Their offsets in the packed buffer are an exclusive scan of the counts; each warp then copies whole lists, so the
        // reads are coalesced and touch only the entries
        const uint32_t cl = threadIdx.x < lists_per_query ? min(list_count[(size_t)blockIdx.x * lists_per_query + threadIdx.x], keep) : 0u;
        uint32_t n_live;
        const uint32_t incl = block_incl_scan(cl, hist + 256, &n_live);
        if (threadIdx.x < lists_per_query) s_off[threadIdx.x] = incl - cl, s_cnt[threadIdx.x] = cl;
        if (threadIdx.x == 0) s_ncomp = n_live;
        __syncthreads();
        if (n_live <= smem_cap) {
            for (uint32_t l = warp; l < lists_per_query; l += kWarps) {
                const uint64_t *src = mine + (size_t)l * keep;
                uint64_t *dst = s_cand + s_off[l];
                for (uint32_t j = lane; j < s_cnt[l]; j += 32) dst[j] = src[j];
            }
        }
    } else {
        for (uint32_t i0 = 0; i0 < total; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const uint64_t c = i < total ? mine[i] : kEmptySlot;
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, c != kEmptySlot);
            uint32_t base = 0;
            if (lane == 0 && m) base = atomicAdd(&s_ncomp, (uint32_t)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            if (c != kEmptySlot) {
                const uint32_t pos = base + __popc(m & ((1u << lane) - 1u));
                if (pos < smem_cap) s_cand[pos] = c;
            }
        }
    }
    __syncthreads();
    const bool packed = s_ncomp <= smem_cap;
    const uint64_t *mine_all = mine; // the proof of the adaptive tier walks the lists as published
    if (packed) total = s_ncomp;
    // candidate i: packed, from shared memory; else from the lists in global memory, where a counted list's slots past its
    // entries are empty
    auto at = [&](uint32_t i) -> uint64_t {
        if (packed) return s_cand[i];
        if (list_count) return i % keep < s_cnt[i / keep] ? mine[i] : kEmptySlot;
        return mine[i];
    };
    // a_k: k-th smallest approximate key; fewer than k candidates: everything survives
    const uint32_t ak_key = block_kth_key(at, total, k, hist, ctl);
    // survivors: approx <= a_k + 2 eps (rounded up)
    const float cut = ak_key == 0xFFFFFFFFu ? __int_as_float(0x7f800000) : key_to_float(ak_key) + (2.0f * eps) * 1.001f + 1e-30f;
    for (uint32_t i0 = 0; i0 < total; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        const uint64_t c = i < total ? at(i) : kEmptySlot;
        const bool take = c != kEmptySlot && (ak_key == 0xFFFFFFFFu || key_to_float((uint32_t)(c >> 32)) <= cut);
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, take);
        uint32_t base = 0;
        if (lane == 0 && m) base = atomicAdd(&s_nsurv, (uint32_t)__popc(m));
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (take) {
            const uint32_t pos = base + __popc(m & ((1u << lane) - 1u));
            if (pos < kSurv) surv[pos] = c;
        }
    }
    __syncthreads();
    const uint32_t n_all = s_nsurv, n_surv = min(n_all, kSurv);
    // Every survivor row is requested at once, one word of each of its 128-byte lines, spread over the block's threads: the
    // rescoring below takes one row per warp and waits on a few rounds of loads per row, each a random row of the corpus (an
    // address translation and an HBM round trip), and these loads have them in flight, or in L2, by then.  The words are only
    // folded into `touch`, which the thread consumes at the very end, so nothing waits for them here
    uint32_t touch = 0;
    {
        const uint32_t row_bytes = dim * (uint32_t)sizeof(float), lines = (row_bytes + 127) / 128;
        for (uint32_t t = threadIdx.x; t < n_surv * lines; t += blockDim.x) {
            const uint8_t *r = rows + (size_t)(uint32_t)surv[t / lines] * pitch;
            touch ^= __ldcg(reinterpret_cast<const uint32_t *>(r + (t % lines) * 128));
        }
    }
    // exact distances of the survivors (one warp per row)
    const uint8_t *qb[1] = {queries + (size_t)q * qpitch};
    for (uint32_t i = warp; i < n_surv; i += kWarps) {
        const uint32_t row = (uint32_t)surv[i];
        const uint8_t *rowb[1] = {rows + (size_t)row * pitch};
        float d[1];
        Tile::run(rowb, qb, dim, lane, d);
        __syncwarp();
        if (lane == 0) surv[i] = make_composite(d[0], kLab ? (uint32_t)row_label[row] : row);
    }
    const uint32_t n_sort = max(32u, next_pow2(n_surv));
    __syncthreads();
    for (uint32_t i = n_surv + threadIdx.x; i < n_sort; i += blockDim.x) surv[i] = kEmptySlot;
    bitonic_sort_smem(surv, n_sort);
    for (uint32_t i = threadIdx.x; i < k; i += blockDim.x) out[(size_t)q * k + i] = i < n_surv ? surv[i] : kEmptySlot;
    // proof
    bool bad = n_all > kSurv; // more candidates within 2 eps of the k-th than the buffer holds: the next tier answers
    // a query whose fp16 form is not finite (row_stats_kernel: |q|^2 = NaN) has no error bound.  And a bound that is not a
    // finite number proves nothing: cut is +-inf or NaN when the k-th approximate key is, or when there are fewer than k
    // candidates; thr_T is +inf when the sample pass found fewer than k finite distances.
    if (q_norm2 && !(q_norm2[blockIdx.x] == q_norm2[blockIdx.x])) bad = true;
    if (!isfinite(cut) || (thr_T && !isfinite(thr_T[blockIdx.x]))) bad = true;
    const bool have_k = n_surv >= k;
    const float ek = have_k ? key_to_float((uint32_t)(surv[k - 1] >> 32)) : 0.0f;
    if (thr_T) {
        if (threadIdx.x == 0 && (overflow[blockIdx.x] != 0 || !have_k || !(thr_T[blockIdx.x] - eps > ek))) bad = true;
    } else {
        for (uint32_t l = threadIdx.x; l < lists_per_query; l += blockDim.x) {
            const uint64_t *lst = mine_all + (size_t)l * keep;
            uint32_t worst = 0;
            bool full = true;
            for (uint32_t j = 0; j < keep; j++) {
                const uint64_t c = lst[j];
                if (c == kEmptySlot)
                    full = false;
                else
                    worst = max(worst, (uint32_t)(c >> 32));
            }
            if (!full) continue; // the list holds every row of its range that passed the kernel's threshold
            if (!have_k)
                bad = true; // fewer than k rows found although a list was truncated
            else if (!(key_to_float(worst) - eps > ek))
                bad = true;
        }
    }
    if (bad) atomicOr(&s_bad, 1u);
    __syncthreads();
    if (threadIdx.x == 0) ok[q] = s_bad ? 0u : ok_value; // 1 = first tier, 2 = second tier (any non-zero = proven)
    asm volatile("" ::"r"(touch));
}

// ------------------------------------------------------------------------------------------------
// Range batches (DESIGN.md §4, "Range queries").  The fixed-bound main pass runs unchanged with the bound
// T[q] = radius[q] + eps_q: a row it drops has approx >= T, so exact >= T - eps_q > radius — it is not in the answer.
// Without a list overflow the kept rows therefore hold every row within the radius, and rescoring them with the exact
// arithmetic of the scan gives the reference's answer.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kRangeWindow = 2048; // list slots packed into shared memory at a time by range_refine_kernel

// T[q] = radius[q] + eps_q, rounded up as threshold_kernel rounds; a radius of +inf or NaN gives a bound that is not
// finite (the main pass keeps everything and the query is never proven).  Also clears the overflow flags and the
// result counter of range_refine_kernel.  One thread per query.
__global__ void range_bound_kernel(const float *__restrict__ radius, uint32_t nq, float eps, const float *__restrict__ q_norm2,
                                   float max_norm, uint32_t dim, int l2, float *__restrict__ thr, uint32_t *__restrict__ overflow,
                                   uint32_t *__restrict__ total) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q == 0) *total = 0;
    if (q >= nq) return;
    const float e = query_eps(eps, q_norm2, q, max_norm, dim, l2 != 0);
    thr[q] = radius[q] + e * 1.001f + 1e-30f;
    overflow[q] = 0;
}

// The direct 16-bit range route (DESIGN.md §4.11): eps16_q bounds |tc - cc| for every stored row and query q, tc = the
// epilogue's 1 - acc of the wgmma pass and cc = the CUDA-core distance (DistTile16).  With mag = sum |x_i q_i| <= M = X |q|
// (X the running maximum row norm) and |e| <= 1 + M for the float64 distance e of the stored values:
//   B_tc = dim 2^-22 M + u (1 + M)                       (DESIGN.md §4, an assumption about the wgmma adder)
//   B_cc = gamma_{m+7} M + u (1 + M) + dim 2^-149        (DESIGN.md §3.1, m = the lane's fmaf chain)
//   eps16_q = 2 (B_tc + B_cc + dim 2^-126)               (2^-126: bf16 products the tensor core may flush from the subnormals)
// evaluated in float64 with every operation rounded up.
constexpr double kR16U = 0x1p-24;         // u, the unit roundoff of fp32
constexpr double kR16TcStep = 0x1p-22;    // B_tc per dimension and unit of M
constexpr double kR16Underflow = 0x1p-149; // B_cc per dimension: fp32 underflow of a product or a partial sum
constexpr double kR16Flush = 0x1p-126;    // per dimension: a product or partial sum flushed to zero by the tensor core
constexpr double kR16Margin = 2.0;        // the factor over B_tc + B_cc
constexpr double kR16MaxMag = 0x1p120;    // M at or above this: never proven (no fp32 overflow in either sum below it)

// One warp per query: |q| from the stored 16-bit query (float64, rounded up), X from max_norm (the float sqrt of the largest
// fp32 |row|^2 row_stats_kernel<DT> found, raised to cover that sum's rounding and underflow), then eps16_q and
// thr[q] = radius[q] + eps16_q rounded up to float.  A query whose |q|, X, M or thr is not finite (or M >= kR16MaxMag) gets
// thr[q] = -inf: the main pass keeps nothing for it and range_refine_kernel never proves it.  Clears overflow[q].
template <int DT>
__global__ void __launch_bounds__(256) range_bound16_kernel(const uint8_t *__restrict__ queries, size_t qpitch, uint32_t nq, uint32_t dim,
                                                            const float *__restrict__ radius, float max_norm, float *__restrict__ thr,
                                                            uint32_t *__restrict__ overflow) {
    const uint32_t q = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    const uint8_t *qb = queries + (size_t)q * qpitch;
    double s = 0.0;
    for (uint32_t i = lane; i < dim; i += 32) {
        const double v = (double)load16<DT>(qb, i);
        s = __fma_ru(v, v, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __dadd_ru(s, __shfl_xor_sync(0xFFFFFFFFu, s, o));
    if (lane != 0) return;
    const double d = (double)dim;
    const double qn = __dsqrt_ru(s);
    // max |row|^2 in fp32: at most dim / 32 + 6 roundings of 2^-24 (<= dim 2^-20 relative) and dim 2^-150 of underflow;
    // sqrtf rounds once more
    const double x = __dadd_ru(__dmul_ru(__dmul_ru((double)max_norm, 1.0 + 0x1p-23), __dsqrt_ru(__fma_ru(d, 0x1p-20, 1.0))),
                               __dsqrt_ru(__dmul_ru(d, 0x1p-149)));
    const double mag = __dmul_ru(x, qn);
    const double chain = 8.0 * ((dim / 8 + 31) / 32) + (double)((dim % 8 + 31) / 32) + 7.0; // m + 7
    const double gamma = __ddiv_ru(chain * kR16U, __dsub_rd(1.0, chain * kR16U));
    const double ue = __dmul_ru(kR16U, __dadd_ru(1.0, mag));                         // u |e|
    const double b_tc = __dadd_ru(__dmul_ru(__dmul_ru(d, kR16TcStep), mag), ue);
    const double b_cc = __dadd_ru(__dadd_ru(__dmul_ru(gamma, mag), ue), __dmul_ru(d, kR16Underflow));
    const double eps = __dmul_ru(kR16Margin, __dadd_ru(__dadd_ru(b_tc, b_cc), __dmul_ru(d, kR16Flush)));
    const float t = __double2float_ru(__dadd_ru((double)radius[q], eps));
    const bool ok = isfinite(qn) && isfinite(x) && mag < kR16MaxMag && isfinite(t);
    thr[q] = ok ? t : -__int_as_float(0x7f800000);
    overflow[q] = 0;
}

// One CTA per query.  Packs the real candidates of the query's `slots` list entries into shared memory a window at a
// time, rescores them from the stored rows (fp32, or 16-bit on the direct route; one warp per row, the scan's own
// arithmetic) and keeps a row iff d <= radius (the reference's inclusive test, brute_force.h range query).  Kept composites are appended to the front
// of the query's own list segment: the count kept so far never exceeds the slots already read, so this overwrites
// only consumed entries.  The segment is then copied to out[off[q], off[q] + cnt[q]) in the dense result buffer, at an
// offset reserved from *total.  ok[q] = 1 unless a list overflowed, the query's fp16 form is not finite (|q|^2 NaN,
// row_stats_kernel) or its bound is not finite; an unproven query writes cnt[q] = 0 and skips the rescoring.
template <int DT, int MT>
__global__ void __launch_bounds__(256) range_refine_kernel(const uint8_t *rows, size_t pitch, uint32_t dim, const uint8_t *queries,
                                                           size_t qpitch, uint32_t slots, uint64_t *cand, const float *__restrict__ radius,
                                                           const float *__restrict__ q_norm2, const float *__restrict__ thr,
                                                           const uint32_t *__restrict__ overflow, uint64_t *__restrict__ out,
                                                           uint32_t *__restrict__ total, uint32_t *__restrict__ ok, uint32_t *__restrict__ cnt,
                                                           uint32_t *__restrict__ off, uint32_t cap) {
    using Tile = DistTile<DT, MT, 1, 1>;
    __shared__ uint64_t s_cand[kRangeWindow];
    __shared__ uint32_t s_n, s_kept, s_base;
    const uint32_t q = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    bool proven = overflow[q] == 0 && isfinite(thr[q]);
    if (q_norm2 && !(q_norm2[q] == q_norm2[q])) proven = false;
    if (!proven) { // the same for every thread of the CTA
        if (threadIdx.x == 0) ok[q] = 0, cnt[q] = 0;
        if (threadIdx.x == 0 && !cap) off[q] = 0;
        return;
    }
    const float r = radius[q];
    uint64_t *mine = cand + (size_t)q * slots;
    const uint8_t *qb[1] = {queries + (size_t)q * qpitch};
    if (threadIdx.x == 0) s_kept = 0;
    for (uint32_t w0 = 0; w0 < slots; w0 += kRangeWindow) {
        const uint32_t wend = min(slots, w0 + kRangeWindow);
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        for (uint32_t i0 = w0; i0 < wend; i0 += blockDim.x) {
            const uint32_t i = i0 + threadIdx.x;
            const uint64_t c = i < wend ? mine[i] : kEmptySlot;
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, c != kEmptySlot);
            uint32_t base = 0;
            if (lane == 0 && m) base = atomicAdd(&s_n, (uint32_t)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            if (c != kEmptySlot) s_cand[base + __popc(m & ((1u << lane) - 1u))] = c;
        }
        __syncthreads();
        const uint32_t n = s_n;
        for (uint32_t i = warp; i < n; i += blockDim.x / 32) {
            const uint32_t row = (uint32_t)s_cand[i];
            const uint8_t *rowb[1] = {rows + (size_t)row * pitch};
            float d[1];
            Tile::run(rowb, qb, dim, lane, d);
            if (lane == 0 && d[0] <= r) mine[atomicAdd(&s_kept, 1u)] = make_composite(d[0], row);
        }
        __syncthreads();
    }
    const uint32_t kept = s_kept;
    if (cap) { // device range batches: the hits into the query's own cap slots, the true count even past cap
        if (threadIdx.x == 0) ok[q] = 1, cnt[q] = kept;
        for (uint32_t i = threadIdx.x; i < min(kept, cap); i += blockDim.x) out[(size_t)q * cap + i] = mine[i];
        return;
    }
    if (threadIdx.x == 0) {
        s_base = atomicAdd(total, kept);
        ok[q] = 1;
        cnt[q] = kept;
        off[q] = s_base;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kept; i += blockDim.x) out[s_base + i] = mine[i];
}

// Fixed-radius pass over 8-bit corpora, one CTA per query: every real entry of its `slots` list entries is a hit with its final
// distance, so they are only packed into out[q][0, cap) (unordered) and counted, the count kept past cap.  ok[q] = 1 unless a
// list overflowed; an overflowed query writes cnt[q] = 0 and nothing else.
__global__ void __launch_bounds__(256) range_pack_kernel(const uint64_t *__restrict__ cand, uint32_t slots, const uint32_t *__restrict__ overflow,
                                                         uint32_t cap, uint64_t *__restrict__ out, uint32_t *__restrict__ cnt,
                                                         uint32_t *__restrict__ ok) {
    __shared__ uint32_t s_n;
    const uint32_t q = blockIdx.x;
    if (overflow[q]) {
        if (threadIdx.x == 0) ok[q] = 0, cnt[q] = 0;
        return;
    }
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const uint64_t *mine = cand + (size_t)q * slots;
    for (uint32_t i = threadIdx.x; i < slots; i += blockDim.x) {
        const uint64_t c = mine[i];
        if (c == kEmptySlot) continue;
        const uint32_t pos = atomicAdd(&s_n, 1u);
        if (pos < cap) out[(size_t)q * cap + pos] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) ok[q] = 1, cnt[q] = s_n;
}

// Device range batches on multi-value indexes (DESIGN.md §4.12), one CTA per query a route proved: its hit rows (the proven
// answer at row level, so every answered label and its best passing row are among them) are mapped to labels, sorted by
// (label, score key, row) in shared memory and the first entry of each label goes to out[q][0, cap) (unordered), counted past
// cap.  front != NULL (fp32 route): the hits are cand[q * slots, + front[q]) of a query with ok[q] != 0; front == NULL (8-bit
// route): the real entries of cand[q * slots, + slots) of a query with overflow[q] == 0.  A proven query with more than
// kRangeFoldMaxHits hits is left open (ok[q] = 0, flags[q] = 3); ok[q] / flags[q] = 1 for a folded query, 0 / 0 for an open one.
// cnt[q] is written for folded queries only.
__global__ void __launch_bounds__(512) range_label_fold_kernel(const uint64_t *__restrict__ cand, uint32_t slots, const uint32_t *__restrict__ front,
                                                               const uint32_t *__restrict__ overflow, const uint64_t *__restrict__ id_to_label,
                                                               uint32_t cap, uint64_t *__restrict__ out, uint32_t *__restrict__ cnt,
                                                               uint32_t *__restrict__ ok, uint32_t *__restrict__ flags) {
    extern __shared__ uint64_t s_hi[]; // (label << 32 | score key) [kRangeFoldMaxHits], then the rows [kRangeFoldMaxHits]
    uint32_t *s_row = reinterpret_cast<uint32_t *>(s_hi + kRangeFoldMaxHits);
    __shared__ uint32_t s_n, s_labels;
    const uint32_t q = blockIdx.x;
    const bool proven = front ? ok[q] != 0 : overflow[q] == 0;
    if (!proven) {
        if (threadIdx.x == 0) ok[q] = 0, flags[q] = 0;
        return;
    }
    const uint64_t *mine = cand + (size_t)q * slots;
    if (threadIdx.x == 0) s_n = 0, s_labels = 0;
    __syncthreads();
    const uint32_t span = front ? front[q] : slots;
    for (uint32_t i = threadIdx.x; i < span; i += blockDim.x) {
        const uint64_t c = mine[i];
        if (c == kEmptySlot) continue;
        const uint32_t pos = atomicAdd(&s_n, 1u);
        if (pos < kRangeFoldMaxHits) {
            s_hi[pos] = (id_to_label[(uint32_t)c] << 32) | (c >> 32); // labels < 2^32 - 1 (the dense label table's rule)
            s_row[pos] = (uint32_t)c;
        }
    }
    __syncthreads();
    const uint32_t n = s_n;
    if (n > kRangeFoldMaxHits) {
        if (threadIdx.x == 0) ok[q] = 0, flags[q] = 3;
        return;
    }
    uint32_t n2 = 1;
    while (n2 < n) n2 <<= 1;
    for (uint32_t i = n + threadIdx.x; i < n2; i += blockDim.x) s_hi[i] = ~0ull, s_row[i] = ~0u; // padding sorts last
    __syncthreads();
    for (uint32_t k = 2; k <= n2; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) {
                const uint32_t p = i ^ j;
                if (p <= i) continue;
                const uint64_t ha = s_hi[i], hb = s_hi[p];
                const uint32_t ra = s_row[i], rb = s_row[p];
                const bool b_first = hb < ha || (hb == ha && rb < ra);
                if (b_first == ((i & k) == 0)) {
                    s_hi[i] = hb, s_hi[p] = ha;
                    s_row[i] = rb, s_row[p] = ra;
                }
            }
            __syncthreads();
        }
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        if (i > 0 && (s_hi[i] >> 32) == (s_hi[i - 1] >> 32)) continue; // not the label's best row
        const uint32_t pos = atomicAdd(&s_labels, 1u);
        if (pos < cap) out[(size_t)q * cap + pos] = (s_hi[i] << 32) | s_row[i];
    }
    __syncthreads();
    if (threadIdx.x == 0) ok[q] = 1, flags[q] = 1, cnt[q] = s_labels;
}

// indices of the queries the first tier left unproven, densely packed: idx[0, *count)
__global__ void compact_unproven_kernel(const uint32_t *__restrict__ ok, uint32_t nq, uint32_t *__restrict__ idx,
                                        uint32_t *__restrict__ count) {
    __shared__ uint32_t n;
    if (threadIdx.x == 0) n = 0;
    __syncthreads();
    for (uint32_t q0 = 0; q0 < nq; q0 += blockDim.x) { // one CTA, ascending order kept chunk by chunk
        const uint32_t q = q0 + threadIdx.x;
        const bool un = q < nq && ok[q] == 0;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, un);
        __shared__ uint32_t wbase[32];
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (lane == 0) wbase[warp] = __popc(m);
        __syncthreads();
        uint32_t before = 0;
        for (int w = 0; w < warp; w++) before += wbase[w];
        uint32_t all = 0;
        for (uint32_t w = 0; w < blockDim.x / 32; w++) all += wbase[w];
        if (un) idx[n + before + __popc(m & ((1u << lane) - 1u))] = q;
        __syncthreads();
        if (threadIdx.x == 0) n += all;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = n;
}
// dst row i = src row idx[i] for i < *count (fp16 query rows and, optionally, their squared norms)
__global__ void gather_queries_kernel(const uint8_t *__restrict__ src, size_t pitch, const float *__restrict__ src_n2,
                                      const uint32_t *__restrict__ idx, const uint32_t *__restrict__ count,
                                      uint8_t *__restrict__ dst, float *__restrict__ dst_n2) {
    const uint32_t n = *count;
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        const uint4 *s4 = reinterpret_cast<const uint4 *>(src + (size_t)idx[i] * pitch);
        uint4 *d4 = reinterpret_cast<uint4 *>(dst + (size_t)i * pitch);
        for (uint32_t c = threadIdx.x; c < pitch / 16; c += blockDim.x) d4[c] = s4[c];
        if (src_n2 && threadIdx.x == 0) dst_n2[i] = src_n2[idx[i]];
    }
}

// ================================================================================================
// host
// ================================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

static bool make_map(CUtensorMap *m, CUtensorMapDataType dt, const void *base, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
                     uint32_t box_inner, uint32_t box_outer) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {pitch_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    return fn(m, dt, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


static constexpr size_t kSmemLimit = 232448; // 227 KB opt-in maximum of dynamic shared memory per CTA on sm_90

template <int V>
static const void *wgmma_kernel_fn_v(CoarseKind kind, uint32_t epl, int epi, int mode, bool filt) {
    if (filt) { // filtered range batches (DESIGN.md §4.13): the 8-bit fixed-radius pass only
        if (kind != CoarseDirect8 || mode != 1) return nullptr;
        if (epi == 2) return (const void *)coarse_wgmma_kernel<true, 8, 4, 1, V, true>;
        return epi == 1 ? (const void *)coarse_wgmma_kernel<true, 8, 2, 1, V, true> : (const void *)coarse_wgmma_kernel<true, 8, 1, 1, V, true>;
    }
    if (kind == CoarseDirect16) {
        if (mode == 1) return (const void *)coarse_wgmma_kernel<true, 8, 0, 1, V>; // fixed bound, lists of 256
        if (mode == 2) return (const void *)coarse_wgmma_kernel<true, 3, 0, 2, V>; // sample pass
        return epl == 3 ? (const void *)coarse_wgmma_kernel<true, 3, 0, 0, V> : (const void *)coarse_wgmma_kernel<true, 8, 0, 0, V>;
    }
    if (kind == CoarseDirect8) {
        if (mode == 1) { // fixed radius (range batches), lists of 256
            if (epi == 2) return (const void *)coarse_wgmma_kernel<true, 8, 4, 1, V>;
            return epi == 1 ? (const void *)coarse_wgmma_kernel<true, 8, 2, 1, V> : (const void *)coarse_wgmma_kernel<true, 8, 1, 1, V>;
        }
        if (epi == 2) return epl == 3 ? (const void *)coarse_wgmma_kernel<true, 3, 4, 0, V> : (const void *)coarse_wgmma_kernel<true, 8, 4, 0, V>;
        if (epi == 1) return epl == 3 ? (const void *)coarse_wgmma_kernel<true, 3, 2, 0, V> : (const void *)coarse_wgmma_kernel<true, 8, 2, 0, V>;
        return epl == 3 ? (const void *)coarse_wgmma_kernel<true, 3, 1, 0, V> : (const void *)coarse_wgmma_kernel<true, 8, 1, 0, V>;
    }
    return nullptr;
}
// K blocks of the resident queries that the fixed-bound pass over the fp16 shadow can hold in registers (16 registers per
// thread each), besides 0: 4 for cosine / inner product with lists of 96 (160 of the launch's 168 registers, no spills).
// The filtered (112 registers without them), squared-L2 (136) and 256-entry-list passes have no room for 64 more and hold none
static constexpr uint32_t kFixedRegKb = 4;
static uint32_t fixed_reg_kb(uint32_t epl, bool l2, bool filt) { return (epl == 3 && !l2 && !filt) ? kFixedRegKb : 0u; }
// variant: 16-bit corpora 1 = bf16, 8-bit corpora 1 = int8 (the fp32 route's shadow is always fp16); epi: CoarseOperands::epilogue
// filt: the kFilt instantiations (fp32 route, where every adaptive-list pass with a filter keeps lists of up to 128; the 8-bit
// fixed-radius pass)
// reg_kb: the fixed-bound pass with that many K blocks of the queries in registers (fixed_reg_kb), else 0
static const void *wgmma_kernel_fn(CoarseKind kind, uint32_t epl, int epi, int mode = 0, uint32_t variant = 0, bool filt = false,
                                   uint32_t reg_kb = 0) {
    const bool l2 = epi != 0;
    if (kind == CoarseDirect16 || kind == CoarseDirect8)
        return variant ? wgmma_kernel_fn_v<1>(kind, epl, epi, mode, filt) : wgmma_kernel_fn_v<0>(kind, epl, epi, mode, filt);
    if (kind == CoarseQ8) { // int8 shadow: fixed bound with lists of 256, the sample pass, adaptive lists of 128 (second tier)
        if (filt || reg_kb || epi) return nullptr;
        if (mode == 1) return (const void *)coarse_wgmma_kernel<false, 8, 5, 1, 1>;
        if (mode == 2) return (const void *)coarse_wgmma_kernel<false, 3, 5, 2, 1>;
        return epl == 8 ? (const void *)coarse_wgmma_kernel<false, 8, 5, 0, 1> : nullptr;
    }
    if (reg_kb) {
        if (mode != 1 || reg_kb != fixed_reg_kb(epl, l2, filt)) return nullptr;
        return (const void *)coarse_wgmma_kernel<false, 3, 0, 1, 0, false, kFixedRegKb>;
    }
    // fp32 route (shadow rows): the flag selects the squared-L2 epilogue; epl 8 = lists of up to 128 (second tier);
    // mode 1 = fixed admission bound (lists of 96, no compaction), mode 2 = the sample pass (slice minima only)
    // (epl 8: lists of 256, k > kCoarseMaxK)
    if (filt) { // hybrid batches: the same passes with the row filter
        if (mode == 1 && epl == 8) return l2 ? (const void *)coarse_wgmma_kernel<false, 8, 3, 1, 0, true> : (const void *)coarse_wgmma_kernel<false, 8, 0, 1, 0, true>;
        if (mode == 1) return l2 ? (const void *)coarse_wgmma_kernel<false, 3, 3, 1, 0, true> : (const void *)coarse_wgmma_kernel<false, 3, 0, 1, 0, true>;
        if (mode == 2) return l2 ? (const void *)coarse_wgmma_kernel<false, 3, 3, 2, 0, true> : (const void *)coarse_wgmma_kernel<false, 3, 0, 2, 0, true>;
        if (epl != 8) return nullptr;
        return l2 ? (const void *)coarse_wgmma_kernel<false, 8, 3, 0, 0, true> : (const void *)coarse_wgmma_kernel<false, 8, 0, 0, 0, true>;
    }
    if (mode == 1 && epl == 8) return l2 ? (const void *)coarse_wgmma_kernel<false, 8, 3, 1> : (const void *)coarse_wgmma_kernel<false, 8, 0, 1>;
    if (mode == 1) return l2 ? (const void *)coarse_wgmma_kernel<false, 3, 3, 1> : (const void *)coarse_wgmma_kernel<false, 3, 0, 1>;
    if (mode == 2) return l2 ? (const void *)coarse_wgmma_kernel<false, 3, 3, 2> : (const void *)coarse_wgmma_kernel<false, 3, 0, 2>;
    if (l2) return epl == 3 ? (const void *)coarse_wgmma_kernel<false, 3, 3, 0> : (const void *)coarse_wgmma_kernel<false, 8, 3, 0>;
    return epl == 3 ? (const void *)coarse_wgmma_kernel<false, 3, 0, 0> : (const void *)coarse_wgmma_kernel<false, 8, 0, 0>;
}
// shared memory of coarse_wgmma_kernel besides the ring: the resident queries (cta_q per CTA, less the reg_kb K blocks held in
// registers), the accumulator transpose (frag: the passes of coarse_frag_epilogue work on the accumulators in registers and
// keep a counter per query instead), the barriers
static size_t wgmma_fixed_smem(uint32_t num_kb, bool frag = false, uint32_t reg_kb = 0, uint32_t cta_q = kQM) {
    return 1024 + (size_t)(num_kb - reg_kb) * cta_q * 128 + (frag ? cta_q * 4 : kQAccBytes) + 2 * kQMaxStages * 8 + 64;
}
static uint32_t wgmma_stages(uint32_t num_kb, bool frag, uint32_t reg_kb, uint32_t cta_q = kQM) {
    return (uint32_t)std::min<size_t>(kQMaxStages, (kSmemLimit - wgmma_fixed_smem(num_kb, frag, reg_kb, cta_q)) / kQStageBytes);
}
// the 16/8-bit kernel needs at least two ring stages next to the resident queries (1024 fp16 dimensions fit)
static bool wgmma_fits_bytes(uint32_t row_bytes, uint32_t cta_q = kQM) {
    return wgmma_fixed_smem(coarse_kb(row_bytes), false, 0, cta_q) + 2 * (size_t)kQStageBytes <= kSmemLimit;
}
static bool wgmma_fits(uint32_t dim) { return wgmma_fits_bytes(dim * 2); }

static size_t fixed_smem(uint32_t num_kb) {
    const uint32_t tn = CfgTF32::kTileN;
    return 1024 + (size_t)num_kb * tn * 128 + (size_t)kTileM * kTF32StageStride * 4 + (size_t)tn * kListCap * 8 + (2 * kMaxStages + 1) * 8 +
           tn * 8 + 64;
}

bool coarse_supported(const CorpusView &c, uint32_t nq, uint32_t k, CoarseKind kind) {
    if (kind == CoarseDirect16) { // fp16 / bf16 corpora, inner product or cosine (normalised rows): tensor-core results are final
        if ((c.dtype != DT_F16 && c.dtype != DT_BF16) || c.metric != MT_IP) return false;
        if (c.dim % 8 != 0 || c.dim < 32 || c.pitch % 16 != 0 || !wgmma_fits(c.dim)) return false;
        if (k > 128 || nq < 1 || c.n_rows < 65536) return false;
        return encode_fn() != nullptr;
    }
    if (kind == CoarseDirect8) { // int8 / uint8 corpora, inner product, cosine or L2: exact integer dot products on s8 / u8 wgmma
        if (c.dtype != DT_I8 && c.dtype != DT_U8) return false;
        if (c.dim % 16 != 0 || c.dim < 32 || c.pitch % 16 != 0 || !wgmma_fits_bytes(c.dim)) return false;
        if (k > 128 || nq < 1 || c.n_rows < 65536) return false;
        return encode_fn() != nullptr;
    }
    if (kind == CoarseQ8) { // fp32 unit rows (the caller checks), inner product on the int8 shadow
        if (c.dtype != DT_F32 || c.metric != MT_IP || c.dim % 8 != 0 || c.dim < 32 || c.dim > 1024 || c.pitch % 16 != 0) return false;
        if (k > kCoarseMaxK || nq < 1 || c.n_rows < 65536 || !wgmma_fits_bytes(c.dim, coarse_cta_queries(true, 1))) return false;
        // rows are padded to whole 256-byte stages: up to 128 dimensions the int8 row streams as many bytes and MMAs as the fp16 one
        if (coarse_kb(c.dim) >= coarse_kb(c.dim * 2)) return false;
        return encode_fn() != nullptr;
    }
    // fp32: cosine / inner product (distance 1 - dot) or squared L2; the caller supplies the error bound (unit vectors or norms)
    if (c.dtype != DT_F32 || (c.metric != MT_IP && c.metric != MT_L2)) return false;
    if (kind == CoarseTF32 && c.metric != MT_IP) return false;
    if (c.dim % 8 != 0 || c.dim < 32 || c.dim > 1024) return false;
    if (c.pitch % 16 != 0) return false;
    // k above kCoarseMaxK: the fp16 route's two-pass first tier only (batch_scan_rows)
    if (k > (kind == CoarseF16 ? kCoarseMaxKWide : kCoarseMaxK) || nq < 1) return false; // batch_scan decides whether a small batch is worth the route
    if (c.n_rows < 65536) return false; // tiny corpora: the exact kernel is already fast
    if (kind == CoarseF16 && !wgmma_fits(c.dim)) return false; // wider rows: the TF32 variant
    if (kind == CoarseTF32 && fixed_smem((c.dim + CfgTF32::kBlockK - 1) / CfgTF32::kBlockK) + 3 * kStageBytes > kSmemLimit) return false;
    return encode_fn() != nullptr;
}

CoarsePlan plan_coarse(const CorpusView &c, uint32_t nq, CoarseKind kind, uint32_t k, uint32_t keep_override, uint32_t tile_stride,
                       int mode, bool filt) {
    CoarsePlan p{};
    p.kind = kind;
    p.tile_stride = std::max(1u, tile_stride);
    // 8-bit corpora: the fixed-radius pass of range batches (mode 1) only
    p.mode = (kind == CoarseF16 || kind == CoarseQ8 || (kind == CoarseDirect16 && c.metric == MT_IP)) ? mode : (kind == CoarseDirect8 && mode == 1) ? 1 : 0;
    if (kind == CoarseF16 || kind == CoarseQ8 || kind == CoarseDirect16 || kind == CoarseDirect8) {
        p.num_kb = coarse_kb(kind == CoarseDirect8 || kind == CoarseQ8 ? c.dim : c.dim * 2);
        p.tiles = ((c.n_rows + kQN - 1) / kQN + p.tile_stride - 1) / p.tile_stride; // row tiles this pass visits
        const uint32_t cta_q = (uint32_t)coarse_cta_queries(kind == CoarseQ8, p.mode);
        p.grid_y = (nq + cta_q - 1) / cta_q;
        const uint32_t sms = (uint32_t)device_sm_count();
        p.grid_x = std::max(1u, std::min(p.tiles, sms / p.grid_y));
        // direct routes: the CTA's exact top-k of its rows.  fp32 route: candidates per (row range, query) — kCoarseKeep
        // for k <= 16, 128 for larger k and for the second tier
        p.keep = (kind == CoarseF16 || kind == CoarseQ8) ? (keep_override ? keep_override : (k <= kCoarseTier1MaxK ? kCoarseKeep : kCoarseKeepWide))
                                   : (k <= 32 ? 32u : 128u);
        p.epl = p.keep <= 32 ? 3 : 8;
        if (p.mode == 1 && kind == CoarseF16) // every row below the bound, up to the list capacity
            p.keep = k > kCoarseMaxK ? kCoarseFixedCapWide : kCoarseFixedCap, p.epl = k > kCoarseMaxK ? 8 : 3;
        if (p.mode == 1 && (kind == CoarseDirect16 || kind == CoarseDirect8)) p.keep = kCoarseFixedCapDirect, p.epl = 8;
        if (p.mode == 1 && kind == CoarseQ8) p.keep = kCoarseFixedCapQ8, p.epl = 8;
        if (p.mode == 2) p.keep = kCoarseSampleSlices, p.epl = 3; // the slice minima
        p.threads = (uint32_t)coarse_threads(kind == CoarseQ8, p.mode);
        const bool frag = coarse_frag_epilogue(kind == CoarseQ8, p.mode);
        const int epi = kind == CoarseQ8 ? 0 : kind == CoarseF16 ? (c.metric == MT_L2 ? 1 : 0) : c.metric == MT_COS ? 1 : (kind == CoarseDirect8 && c.metric == MT_L2) ? 2 : 0;
        // the fixed-bound pass over the shadow holds the leading K blocks of its queries in registers where that frees shared
        // memory for one more ring stage and leaves at least one stage of queries in shared memory
        static int rcap = -1; // VECSIM_B200_REGKB caps the register-held K blocks (0 = none)
        if (rcap < 0) {
            const char *e = getenv("VECSIM_B200_REGKB");
            rcap = e ? std::max(0, atoi(e)) : (int)kFixedRegKb;
        }
        p.reg_kb = 0;
        if (kind == CoarseF16 && p.mode == 1) {
            const uint32_t rk = fixed_reg_kb(p.epl, epi != 0, filt);
            if (rk && (int)rk <= rcap && p.num_kb >= rk + kQKbPerStage && wgmma_stages(p.num_kb, frag, rk) > wgmma_stages(p.num_kb, frag, 0))
                p.reg_kb = rk;
        }
        p.stages = wgmma_stages(p.num_kb, frag, p.reg_kb, cta_q);
        p.smem_bytes = wgmma_fixed_smem(p.num_kb, frag, p.reg_kb, cta_q) + (size_t)p.stages * kQStageBytes;
        // the query groups of a row range form a thread-block cluster (multicast of the row tiles).  128 queries per CTA: pairs at
        // most, which can fill all 132 SMs where clusters of four leave 12 idle (DESIGN.md §4.2)
        p.csize = 1;
        static int ccap = -1; // VECSIM_B200_CLUSTER caps the cluster size (1 = no clusters)
        if (ccap < 0) {
            const char *e = getenv("VECSIM_B200_CLUSTER");
            ccap = e ? std::max(1, atoi(e)) : 4;
        }
        for (uint32_t cs = cta_q > kQM ? 2 : 4; cs > 1; cs >>= 1)
            if ((int)cs <= ccap && p.grid_y % cs == 0 && (kQStageBytes / kQKbPerStage) % (16 * cs) == 0) {
                p.csize = cs;
                break;
            }
        const void *kfn = wgmma_kernel_fn(kind, p.epl, epi, p.mode, (c.dtype == DT_BF16 || c.dtype == DT_I8 || kind == CoarseQ8) ? 1u : 0u, filt,
                                          p.reg_kb);
        if (p.csize > 1) {
            cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem_bytes);
            cudaLaunchConfig_t cfg{};
            cudaLaunchAttribute at[1];
            cfg.gridDim = dim3(1, p.grid_y, 1);
            cfg.blockDim = dim3(p.threads); // a block size the kernel cannot take reports no cluster: csize would fall to 1
            cfg.dynamicSmemBytes = p.smem_bytes;
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = 1, at[0].val.clusterDim.y = p.csize, at[0].val.clusterDim.z = 1;
            cfg.attrs = at, cfg.numAttrs = 1;
            int nclusters = 0;
            if (cudaOccupancyMaxActiveClusters(&nclusters, kfn, &cfg) != cudaSuccess || nclusters < 1) {
                cudaGetLastError();
                p.csize = 1;
            } else {
                // one wave of co-resident clusters: grid_x row ranges x (grid_y / csize) clusters each
                p.grid_x = std::max(1u, std::min(p.grid_x, (uint32_t)nclusters / (p.grid_y / p.csize)));
            }
        }
        p.cand_elems = (size_t)nq * p.grid_x * p.keep;
        p.scratch_elems = (size_t)p.grid_x * p.grid_y * (p.epl * 32) * kQListStride;
        return p;
    }
    const uint32_t bk = CfgTF32::kBlockK, tn = CfgTF32::kTileN;
    p.num_kb = (c.dim + bk - 1) / bk;
    p.tiles = (c.n_rows + kTileM - 1) / kTileM;
    p.grid_y = (nq + tn - 1) / tn;
    const uint32_t sms = (uint32_t)device_sm_count();
    p.grid_x = std::max(1u, std::min(p.tiles, sms / p.grid_y));
    p.keep = kCoarseKeep;
    const size_t fixed_bytes = fixed_smem(p.num_kb);
    p.threads = kCoarseThreads;
    p.stages = (uint32_t)std::min<size_t>(kMaxStages, (kSmemLimit - fixed_bytes) / kStageBytes);
    p.cand_elems = (size_t)nq * p.grid_x * p.keep;
    p.smem_bytes = fixed_bytes + (size_t)p.stages * kStageBytes;
    return p;
}

template <class Cfg>
static cudaError_t launch_coarse_t(const void *rows, size_t pitch, uint32_t n_rows, uint32_t dim, const void *d_queries, size_t qpitch,
                                   uint32_t nq, const CoarsePlan &p, uint64_t *d_cand, cudaStream_t s) {
    const CUtensorMapDataType dt = Cfg::kElem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    CUtensorMap ma, mq;
    if (!make_map(&ma, dt, rows, dim, n_rows, pitch, Cfg::kBlockK, kTileM)) return cudaErrorInvalidValue;
    if (!make_map(&mq, dt, d_queries, dim, nq, qpitch, Cfg::kBlockK, Cfg::kTileN)) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(coarse_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem_bytes);
    if (e != cudaSuccess) return e;
    coarse_kernel<Cfg><<<dim3(p.grid_x, p.grid_y), p.threads, p.smem_bytes, s>>>(ma, mq, n_rows, nq, p.num_kb, p.tiles, p.keep, p.stages,
                                                                                d_cand);
    return cudaGetLastError();
}

cudaError_t launch_coarse(const CoarseOperands &o, uint32_t n_rows, uint32_t dim, uint32_t nq, const CoarsePlan &p, uint64_t *d_cand,
                          uint64_t *d_scratch, cudaStream_t s, const uint32_t *d_nq_dev, const float *d_thr_fixed, uint32_t *d_overflow,
                          const uint32_t *d_filt, uint32_t filt_words, const uint32_t *d_filt_q, uint32_t *d_list_count) {
    if (d_filt && p.kind != CoarseF16 && !(p.kind == CoarseDirect8 && p.mode == 1)) return cudaErrorInvalidValue;
    if (p.kind == CoarseF16 || p.kind == CoarseQ8 || p.kind == CoarseDirect16 || p.kind == CoarseDirect8) {
        if (p.mode == 1 && (!d_thr_fixed || !d_overflow)) return cudaErrorInvalidValue;
        if (p.mode == 1 && p.kind == CoarseQ8 && !d_list_count) return cudaErrorInvalidValue; // its lists are not padded
        // operand variant: 16-bit 1 = bf16 (else fp16); 8-bit 1 = int8 (else uint8); the fp16 shadow of the fp32 route: 0
        const uint32_t ev = (p.kind == CoarseDirect16 || p.kind == CoarseDirect8) && o.elem_variant ? 1u : 0u;
        const void *kfn = wgmma_kernel_fn(p.kind, p.epl, o.epilogue, p.mode, ev, d_filt != nullptr, p.reg_kb);
        if (!kfn) return cudaErrorInvalidValue;
        cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem_bytes);
        if (e != cudaSuccess) {
            fprintf(stderr, "vecsim_b200: coarse pass: %zu bytes of shared memory refused: %s\n", p.smem_bytes, cudaGetErrorString(e));
            return e;
        }
        CUtensorMap mr{};
        uint32_t row_bytes = dim * 2;
        if (p.kind == CoarseDirect16) {
            if (!make_map(&mr, ev ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, o.rows, dim, n_rows, o.pitch, 64,
                          kQN / p.csize))
                return cudaErrorInvalidValue;
        } else if (p.kind == CoarseQ8) {
            row_bytes = (uint32_t)coarse_q8_payload(dim); // the query's scale follows its payload
        } else if (p.kind == CoarseDirect8) {
            row_bytes = dim;
            if (!make_map(&mr, CU_TENSOR_MAP_DATA_TYPE_UINT8, o.rows, dim, n_rows, o.pitch, 128, kQN / p.csize)) return cudaErrorInvalidValue;
        }
        cudaLaunchConfig_t cfg{};
        cudaLaunchAttribute at[1];
        cfg.gridDim = dim3(p.grid_x, p.grid_y, 1);
        cfg.blockDim = dim3(p.threads);
        cfg.dynamicSmemBytes = p.smem_bytes;
        cfg.stream = s;
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = 1, at[0].val.clusterDim.y = p.csize, at[0].val.clusterDim.z = 1;
        cfg.attrs = at, cfg.numAttrs = 1;
        const uint8_t *rows = static_cast<const uint8_t *>(o.rows), *qs = static_cast<const uint8_t *>(o.queries);
        size_t rp = o.pitch, qp = o.qpitch;
        const float *rn2 = o.row_norm2, *qn2 = o.q_norm2;
        uint32_t a_nrows = n_rows, a_nq = nq, a_dim = dim, a_rb = row_bytes, a_kb = p.num_kb, a_tiles = p.tiles, a_keep = p.keep,
                 a_st = p.stages, a_cs = p.csize, a_stride = p.tile_stride;
        void *args[] = {&mr,   &rows,    &rp,     &qs,   &qp,   &rn2,  &qn2,      &a_nrows, &a_nq,     &a_dim,       &a_rb, &a_kb,
                        &a_tiles, &a_keep, &a_st, &a_cs, &d_scratch, &d_cand, &d_nq_dev, &a_stride, &d_thr_fixed, &d_overflow,
                        &d_filt, &filt_words, &d_filt_q, &d_list_count};
        const cudaError_t le = cudaLaunchKernelExC(&cfg, kfn, args);
        if (le != cudaSuccess)
            fprintf(stderr, "vecsim_b200: coarse pass launch failed (kind %d mode %d csize %u grid %u x %u smem %zu): %s\n", (int)p.kind,
                    p.mode, p.csize, p.grid_x, p.grid_y, p.smem_bytes, cudaGetErrorString(le));
        return le;
    }
    return launch_coarse_t<CfgTF32>(o.rows, o.pitch, n_rows, dim, o.queries, o.qpitch, nq, p, d_cand, s);
}

#ifdef COARSE_CYCLE_ACCOUNT
// the cycle account of the last fixed-bound pass, [cta][role][kCaSlots] as unsigned 64-bit, into host memory; returns
// the slots per (cta, role)
extern "C" int VecSimB200_CoarseCycles(unsigned long long *host, int max_ctas) {
    const size_t bytes = (size_t)std::min(max_ctas, kCaMaxCtas) * 3 * kCaSlots * sizeof(unsigned long long);
    if (cudaMemcpyFromSymbol(host, g_coarse_cycles, bytes) != cudaSuccess) return -1;
    return kCaSlots;
}
#endif

// fp32 rows -> the tiled fp16 shadow: [tile of 128 rows][K block of 64 halves][128 rows x 128 B, 128B-swizzled],
// i.e. exactly the bytes a SWIZZLE_128B tensor-map load would have produced in shared memory, so that
// coarse_wgmma_kernel can stream it with contiguous bulk copies.  One 16-byte chunk (8 halves) per thread;
// chunks past `dim` are zero.
__global__ void __launch_bounds__(256) to_f16_tiled_kernel(const uint8_t *__restrict__ src, size_t spitch, uint32_t dim, uint32_t first,
                                                           uint32_t n, uint8_t *__restrict__ dst, uint32_t num_kb) {
    const uint32_t per_row = num_kb * 8;
    const size_t total = (size_t)n * per_row;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t r = first + (uint32_t)(i / per_row), ci = (uint32_t)(i % per_row);
        uint4 o = make_uint4(0, 0, 0, 0);
        if (ci * 8 < dim) {
            const float4 *p = reinterpret_cast<const float4 *>(src + (size_t)r * spitch) + 2 * ci;
            const float4 x = p[0], y = p[1];
            __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
            __half2 h2 = __floats2half2_rn(y.x, y.y), h3 = __floats2half2_rn(y.z, y.w);
            o.x = *reinterpret_cast<uint32_t *>(&h0);
            o.y = *reinterpret_cast<uint32_t *>(&h1);
            o.z = *reinterpret_cast<uint32_t *>(&h2);
            o.w = *reinterpret_cast<uint32_t *>(&h3);
        }
        const uint32_t tile = r / kQN, rr = r % kQN, kb = ci / 8, c = ci % 8;
        uint8_t *blk = dst + ((size_t)tile * num_kb + kb) * kQBlockBytes;
        *reinterpret_cast<uint4 *>(blk + rr * 128 + ((c ^ (rr & 7)) * 16)) = o;
    }
}

size_t coarse_shadow_bytes(uint32_t rows, uint32_t dim) {
    return (size_t)((rows + kQN - 1) / kQN) * coarse_kb(dim * 2) * kQBlockBytes;
}

cudaError_t launch_to_f16_tiled(const void *src, size_t spitch, uint32_t dim, uint32_t first, uint32_t n, void *dst, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const uint32_t num_kb = coarse_kb(dim * 2);
    const size_t total = (size_t)n * num_kb * 8;
    const uint32_t grid = (uint32_t)std::max<size_t>(1, std::min<size_t>((total + 255) / 256, (size_t)device_sm_count() * 16));
    to_f16_tiled_kernel<<<grid, 256, 0, s>>>(static_cast<const uint8_t *>(src), spitch, dim, first, n, static_cast<uint8_t *>(dst), num_kb);
    return cudaGetLastError();
}

// fp32 unit rows -> the tiled int8 shadow: [tile of 128 rows][K block of 128 int8][128 rows x 128 B, 128B-swizzled], the image
// of to_f16_tiled_kernel with one-byte elements.  One CTA per tile: the tile's max |x| gives its scale s_t = max / 127 (1 for an
// all-zero tile, so that no scale is 0), every element x becomes rint(x / s_t) (|x / s_t| <= 127 up to rounding, clamped), rows
// past n_rows and bytes past dim are zero.  The residual norm |x - s_t x~| and the norm |x| of each row are accumulated in fp64
// and folded, rounded up to float, into the running maxima stats[0] and stats[1] (as bits: the values are >= 0; a NaN or inf
// element makes them NaN / inf, and the host keeps such an index off the route).
__global__ void __launch_bounds__(256) to_i8_tiled_kernel(const uint8_t *__restrict__ src, size_t spitch, uint32_t dim, uint32_t n_rows,
                                                          uint32_t tile0, uint32_t ntiles, uint8_t *__restrict__ dst, uint32_t num_kb,
                                                          float *__restrict__ tscale, uint32_t *__restrict__ stats) {
    __shared__ float s_max[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float w_res = 0.0f, w_nrm = 0.0f; // this warp's maxima over its rows
    for (uint32_t t = tile0 + blockIdx.x; t < tile0 + ntiles; t += gridDim.x) {
        float m = 0.0f;
        for (uint32_t rr = warp; rr < (uint32_t)kQN; rr += 8) {
            const uint32_t r = t * kQN + rr;
            if (r >= n_rows) break;
            const float *x = reinterpret_cast<const float *>(src + (size_t)r * spitch);
            for (uint32_t e = lane * 4; e < dim; e += 128) {
                const float4 v = *reinterpret_cast<const float4 *>(x + e);
                m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
                if (!(v.x == v.x && v.y == v.y && v.z == v.z && v.w == v.w)) m = __int_as_float(0x7f800000);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
        if (lane == 0) s_max[warp] = m;
        __syncthreads();
        m = s_max[0];
        for (int w = 1; w < 8; w++) m = fmaxf(m, s_max[w]);
        __syncthreads(); // s_max is rewritten by the next tile
        const float sc = m > 0.0f ? __fdiv_rn(m, 127.0f) : 1.0f;
        if (threadIdx.x == 0) tscale[t] = sc;
        for (uint32_t rr = warp; rr < (uint32_t)kQN; rr += 8) {
            const uint32_t r = t * kQN + rr;
            const bool real = r < n_rows;
            const float *x = reinterpret_cast<const float *>(src + (size_t)(real ? r : 0) * spitch);
            double res2 = 0.0, nrm2 = 0.0;
            for (uint32_t ci = lane; ci < num_kb * 8; ci += 32) { // 16-element chunk ci of the row
                uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int g = 0; g < 4; g++) {
                    const uint32_t e = ci * 16 + g * 4;
                    if (!real || e >= dim) continue; // dim % 8 == 0: a float4 is all in or all out
                    const float4 v = *reinterpret_cast<const float4 *>(x + e);
                    const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int h = 0; h < 4; h++) {
                        const float qv = fminf(fmaxf(rintf(__fdiv_rn(f[h], sc)), -127.0f), 127.0f);
                        const double d = (double)f[h] - (double)sc * (double)qv;
                        res2 = fma(d, d, res2);
                        nrm2 = fma((double)f[h], (double)f[h], nrm2);
                        w[g] |= ((uint32_t)(int)qv & 0xFFu) << (8 * h);
                    }
                }
                const uint32_t kb = ci / 8, c = ci % 8;
                uint8_t *blk = dst + ((size_t)t * num_kb + kb) * kQBlockBytes;
                *reinterpret_cast<uint4 *>(blk + rr * 128 + ((c ^ (rr & 7)) * 16)) = make_uint4(w[0], w[1], w[2], w[3]);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                res2 += __shfl_xor_sync(0xFFFFFFFFu, res2, o);
                nrm2 += __shfl_xor_sync(0xFFFFFFFFu, nrm2, o);
            }
            const float rn = __double2float_ru(sqrt(res2));
            w_res = (rn == rn && w_res == w_res) ? fmaxf(w_res, rn) : __int_as_float(0x7fc00000); // a NaN sticks
            w_nrm = fmaxf(w_nrm, __double2float_ru(sqrt(nrm2)));
        }
    }
    if (lane == 0) { // NaN has a larger bit pattern than any non-negative float: it wins the maximum
        atomicMax(&stats[0], __float_as_uint(w_res));
        atomicMax(&stats[1], __float_as_uint(w_nrm));
    }
}

size_t coarse_shadow8_bytes(uint32_t rows, uint32_t dim) {
    return (size_t)((rows + kQN - 1) / kQN) * coarse_kb(dim) * kQBlockBytes;
}

cudaError_t launch_to_i8_tiled(const void *src, size_t spitch, uint32_t dim, uint32_t n_rows, uint32_t first, uint32_t n, void *dst,
                               float *d_tscale, uint32_t *d_stats, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    if (dim % 8 != 0 || spitch % 16 != 0) return cudaErrorInvalidValue;
    const uint32_t tile0 = first / kQN, ntiles = (first + n - 1) / kQN - tile0 + 1;
    const uint32_t grid = std::max(1u, std::min(ntiles, (uint32_t)device_sm_count() * 8));
    to_i8_tiled_kernel<<<grid, 256, 0, s>>>(static_cast<const uint8_t *>(src), spitch, dim, n_rows, tile0, ntiles, static_cast<uint8_t *>(dst),
                                            coarse_kb(dim), d_tscale, d_stats);
    return cudaGetLastError();
}

// One warp per fp32 unit query q: its scale s_q = max |q_i| / 127 (1 for a zero query), q~ = rint(q / s_q) into the int8 row
// (zero padded to the payload), s_q after the payload, and the bound of |approx - exact| for every stored row x:
//   q.x - s_q s_t q~.x~ = q.delta + eta.x - eta.delta   (x = s_t x~ + delta, q = s_q q~ + eta)
//   |.| <= |q| delta_max + |eta| x_max + |eta| delta_max                        (Cauchy-Schwarz)
// plus the fp32 rounding of both sides: the exact scan's dot product (at most dim 2^-24 |q| |x| in any order) and the approximate
// distance 1 - fl(fl(s_q s_t) acc) (two roundings of a value below (|q| + |eta|)(x_max + delta_max), one of 1 - it), all
// covered by (dim + 8) 2^-23 (|q| + |eta|)(x_max + delta_max) + 2^-21; the sum is computed in fp64 and rounded up.  A query whose
// bound is not finite gets NaN, which refine_kernel never proves.
__global__ void __launch_bounds__(256) quantize_queries_kernel(const uint8_t *__restrict__ q, size_t qpitch, uint32_t dim, uint32_t nq,
                                                               uint8_t *__restrict__ q8, size_t pitch8, uint32_t payload,
                                                               float *__restrict__ eps, float delta_max, float x_max) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * 8 + warp;
    if (i >= nq) return;
    const float *x = reinterpret_cast<const float *>(q + (size_t)i * qpitch);
    float m = 0.0f;
    bool finite = true;
    for (uint32_t e = lane; e < dim; e += 32) {
        const float v = x[e];
        m = fmaxf(m, fabsf(v));
        finite = finite && fabsf(v) <= 3.4e38f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
    finite = __all_sync(0xFFFFFFFFu, finite);
    const float sc = (finite && m > 0.0f) ? __fdiv_rn(m, 127.0f) : 1.0f;
    double qn2 = 0.0, en2 = 0.0;
    uint8_t *dst = q8 + (size_t)i * pitch8;
    for (uint32_t e = lane; e < payload; e += 32) {
        int8_t b = 0;
        if (e < dim && finite) {
            const float v = x[e];
            const float qv = fminf(fmaxf(rintf(__fdiv_rn(v, sc)), -127.0f), 127.0f);
            const double d = (double)v - (double)sc * (double)qv;
            en2 = fma(d, d, en2);
            qn2 = fma((double)v, (double)v, qn2);
            b = (int8_t)(int)qv;
        }
        dst[e] = (uint8_t)b;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        qn2 += __shfl_xor_sync(0xFFFFFFFFu, qn2, o);
        en2 += __shfl_xor_sync(0xFFFFFFFFu, en2, o);
    }
    if (lane == 0) {
        *reinterpret_cast<float *>(dst + payload) = sc;
        const double qn = sqrt(qn2), en = sqrt(en2), X = (double)x_max, D = (double)delta_max;
        double e = qn * D + en * X + en * D + (double)(dim + 8) * 0x1p-23 * (qn + en) * (X + D) + 0x1p-21;
        e *= 1.0001;
        const float ef = __double2float_ru(e);
        eps[i] = (finite && isfinite(ef)) ? ef : __int_as_float(0x7fc00000);
    }
}

cudaError_t launch_quantize_queries(const void *d_q, size_t qpitch, uint32_t dim, uint32_t nq, void *d_q8, float *d_eps, float delta_max,
                                    float x_max, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    quantize_queries_kernel<<<(nq + 7) / 8, 256, 0, s>>>(static_cast<const uint8_t *>(d_q), qpitch, dim, nq, static_cast<uint8_t *>(d_q8),
                                                         coarse_q8_pitch(dim), (uint32_t)coarse_q8_payload(dim), d_eps, delta_max, x_max);
    return cudaGetLastError();
}

// squared norm of fp32 rows [first, first+n) -> norm2[first + r]; running maxima (as float bits: the values are >= 0,
// a NaN compares as huge and disables the route) of the squared norm and of |x| into stats[0], stats[1].
// A row (in practice a query: rows outside the fp16 range keep their index off the route) whose fp16 form is not finite
// — a component with |x| >= 65520 rounds to inf, or is NaN — gets norm2 = NaN: its approximate distances are inf or NaN,
// query_eps does not bound them, and refine_kernel never proves such a query.
// DT_F16 / DT_BF16: the stored 16-bit rows of the direct range route (DESIGN.md §4.11), which reads only the running maximum of
// the squared norm (a NaN or inf component makes it NaN or inf, and the route then leaves the batch to the exact scan).
template <int DT>
__global__ void __launch_bounds__(256) row_stats_kernel(const uint8_t *__restrict__ rows, size_t pitch, uint32_t dim, uint32_t first,
                                                        uint32_t n, float *__restrict__ norm2, uint32_t *__restrict__ stats) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t r = blockIdx.x * 8 + warp; r < n; r += gridDim.x * 8) {
        const uint8_t *x = rows + (size_t)(first + r) * pitch;
        float s = 0.0f, m = 0.0f;
        for (uint32_t i = lane; i < dim; i += 32) {
            const float v = DT == DT_F32 ? reinterpret_cast<const float *>(x)[i] : load16<DT>(x, i);
            s = fmaf(v, v, s);
            m = fmaxf(m, fabsf(v));
            if (v != v) m = __int_as_float(0x7f800000);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
            m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
        }
        if (lane == 0) {
            norm2[first + r] = m < 65520.0f ? s : __int_as_float(0x7fc00000);
            if (stats) {
                atomicMax(&stats[0], __float_as_uint(s));
                atomicMax(&stats[1], __float_as_uint(m));
            }
        }
    }
}
cudaError_t launch_row_stats(const void *rows, size_t pitch, uint32_t dim, uint32_t first, uint32_t n, float *d_norm2, uint32_t *d_stats,
                             cudaStream_t s, int dtype) {
    if (n == 0) return cudaSuccess;
    const uint32_t grid = std::max(1u, std::min((n + 7) / 8, (uint32_t)device_sm_count() * 8));
    const uint8_t *r = static_cast<const uint8_t *>(rows);
    if (dtype == DT_F32)
        row_stats_kernel<DT_F32><<<grid, 256, 0, s>>>(r, pitch, dim, first, n, d_norm2, d_stats);
    else if (dtype == DT_F16)
        row_stats_kernel<DT_F16><<<grid, 256, 0, s>>>(r, pitch, dim, first, n, d_norm2, d_stats);
    else if (dtype == DT_BF16)
        row_stats_kernel<DT_BF16><<<grid, 256, 0, s>>>(r, pitch, dim, first, n, d_norm2, d_stats);
    else
        return cudaErrorInvalidValue;
    return cudaGetLastError();
}

// exact int32 squared norm of int8 / uint8 rows [first, first+n) -> norm2[first + r]; one warp per row, 16 bytes per lane
// and step (dim % 16 == 0, pitch % 16 == 0).  At most 65025 * 2048 < 2^31.
template <bool kSigned>
__global__ void __launch_bounds__(256) int_norm2_kernel(const uint8_t *__restrict__ rows, size_t pitch, uint32_t dim, uint32_t first,
                                                        uint32_t n, int32_t *__restrict__ norm2) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t r = blockIdx.x * 8 + warp; r < n; r += gridDim.x * 8) {
        const uint8_t *x = rows + (size_t)(first + r) * pitch;
        int s = 0;
        for (uint32_t i = lane * 16; i < dim; i += 32 * 16) {
            const uint4 w = *reinterpret_cast<const uint4 *>(x + i);
            const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int t = 0; t < 4; t++) s = kSigned ? __dp4a((int)u[t], (int)u[t], s) : (int)__dp4a(u[t], u[t], (uint32_t)s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
        if (lane == 0) norm2[first + r] = s;
    }
}
cudaError_t launch_int_norm2(const void *rows, size_t pitch, uint32_t dim, uint32_t first, uint32_t n, bool is_signed, int32_t *d_norm2,
                             cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    if (dim % 16 != 0 || pitch % 16 != 0 || dim > 2048) return cudaErrorInvalidValue;
    const uint32_t grid = std::max(1u, std::min((n + 7) / 8, (uint32_t)device_sm_count() * 8));
    const uint8_t *r = static_cast<const uint8_t *>(rows);
    if (is_signed)
        int_norm2_kernel<true><<<grid, 256, 0, s>>>(r, pitch, dim, first, n, d_norm2);
    else
        int_norm2_kernel<false><<<grid, 256, 0, s>>>(r, pitch, dim, first, n, d_norm2);
    return cudaGetLastError();
}

cudaError_t launch_to_f16(const void *src, size_t spitch, uint32_t dim, uint32_t first, uint32_t n, void *dst, size_t dpitch,
                          cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const size_t total = (size_t)n * (dim / 8);
    const uint32_t grid = (uint32_t)std::max<size_t>(1, std::min<size_t>((total + 255) / 256, (size_t)device_sm_count() * 16));
    to_f16_kernel<<<grid, 256, 0, s>>>(static_cast<const uint8_t *>(src), spitch, dim, first, n, static_cast<uint8_t *>(dst), dpitch);
    return cudaGetLastError();
}

cudaError_t launch_refine(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t lists_per_query, uint32_t keep,
                          uint32_t k, const uint64_t *d_cand, float eps, const float *d_q_norm2, float max_norm, uint32_t *d_ok,
                          uint64_t *d_out, const uint32_t *d_q_index, const uint32_t *d_nq_dev, cudaStream_t s, const float *d_thr_T,
                          const uint32_t *d_overflow, const uint64_t *d_row_label, const float *d_q_eps, const uint32_t *d_list_count) {
    if (nq == 0) return cudaSuccess;
    const uint32_t okv = d_q_index ? 2u : 1u;
    const uint8_t *rows = static_cast<const uint8_t *>(c.rows), *qs = static_cast<const uint8_t *>(d_queries);
    // candidates packed in shared memory: as many slots as the lists have, up to 20 KB worth (k > kCoarseMaxK: 64 KB, two CTAs
    // per SM next to the 32 KB survivor buffer; counted lists: 64 KB)
    const bool wide = k > kCoarseMaxK;
    if (k > kCoarseMaxKWide) return cudaErrorInvalidValue;
    if (d_list_count && (!d_thr_T || lists_per_query > kRefineMaxLists)) return cudaErrorInvalidValue;
    const uint32_t max_cap = wide ? kRefineCapWide : d_list_count ? kRefineCapCounted : kRefineCapPadded;
    const uint32_t smem_cap = std::min<uint32_t>(lists_per_query * keep, max_cap);
    const size_t smem = (size_t)smem_cap * 8;
    const auto kern = d_row_label ? (c.metric == MT_L2 ? (wide ? refine_kernel<MT_L2, kRefineMaxSurvWide, true> : refine_kernel<MT_L2, kRefineMaxSurv, true>)
                                                      : (wide ? refine_kernel<MT_IP, kRefineMaxSurvWide, true> : refine_kernel<MT_IP, kRefineMaxSurv, true>))
                    : c.metric == MT_L2 ? (wide ? refine_kernel<MT_L2, kRefineMaxSurvWide> : refine_kernel<MT_L2, kRefineMaxSurv>)
                                        : (wide ? refine_kernel<MT_IP, kRefineMaxSurvWide> : refine_kernel<MT_IP, kRefineMaxSurv>);
    // the 48 KB a launch gets without opting in cover static + dynamic shared memory (the wide survivor buffer alone is 32 KB).
    // Opt in to the largest packing any launch of an instantiation can ask for, the same value every time: concurrent launches
    // of the same kernel from other host threads never see the limit lowered under them
    constexpr uint32_t kOptIn = std::max(kRefineCapWide, kRefineCapCounted) * 8;
    cudaFuncAttributes fa{};
    cudaError_t e = cudaFuncGetAttributes(&fa, kern);
    if (e != cudaSuccess) return e;
    if (fa.sharedSizeBytes + smem > 48 * 1024 && fa.maxDynamicSharedSizeBytes < (int)kOptIn) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kOptIn);
        if (e != cudaSuccess) return e;
    }
    kern<<<nq, kRefineThreads, smem, s>>>(rows, c.pitch, c.dim, qs, qpitch, nq, lists_per_query, keep, k, d_cand, eps, d_q_norm2, max_norm, d_ok, okv,
                               d_out, d_q_index, d_nq_dev, d_thr_T, d_overflow, smem_cap, d_row_label, d_q_eps, d_list_count);
    return cudaGetLastError();
}

cudaError_t launch_threshold(const uint64_t *d_cand, uint32_t nq, uint32_t lists_per_query, uint32_t keep, uint32_t k, float eps,
                             const float *d_q_norm2, float max_norm, uint32_t dim, int l2, float *d_thr, uint32_t *d_overflow, cudaStream_t s,
                             const float *d_q_eps) {
    if (nq == 0) return cudaSuccess;
    threshold_kernel<<<nq, 256, 0, s>>>(d_cand, nq, lists_per_query, keep, k, eps, d_q_norm2, max_norm, dim, l2, d_thr, d_overflow, d_q_eps);
    return cudaGetLastError();
}

__global__ void flags_from_overflow_kernel(const uint32_t *__restrict__ ovf, uint32_t nq, uint32_t *__restrict__ ok) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq) ok[q] = ovf[q] ? 0u : 1u;
}
cudaError_t launch_flags_from_overflow(const uint32_t *d_overflow, uint32_t nq, uint32_t *d_ok, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    flags_from_overflow_kernel<<<(nq + 255) / 256, 256, 0, s>>>(d_overflow, nq, d_ok);
    return cudaGetLastError();
}
__global__ void scatter_rows_kernel(const uint64_t *__restrict__ src, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ count,
                                    uint32_t k, uint64_t *__restrict__ dst, uint32_t *__restrict__ ok) {
    const uint32_t n = *count;
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        const uint32_t q = idx[i];
        for (uint32_t t = threadIdx.x; t < k; t += blockDim.x) dst[(size_t)q * k + t] = src[(size_t)i * k + t];
        if (threadIdx.x == 0) ok[q] = 2u;
    }
}
cudaError_t launch_scatter_rows(const uint64_t *d_src, const uint32_t *d_idx, const uint32_t *d_count, uint32_t max_n, uint32_t k,
                                uint64_t *d_dst, uint32_t *d_ok, cudaStream_t s) {
    if (max_n == 0) return cudaSuccess;
    scatter_rows_kernel<<<std::min(max_n, 256u), 128, 0, s>>>(d_src, d_idx, d_count, k, d_dst, d_ok);
    return cudaGetLastError();
}

cudaError_t launch_compact_unproven(const uint32_t *d_ok, uint32_t nq, uint32_t *d_idx, uint32_t *d_count, cudaStream_t s) {
    compact_unproven_kernel<<<1, 256, 0, s>>>(d_ok, nq, d_idx, d_count);
    return cudaGetLastError();
}
cudaError_t launch_range_bound(const float *d_radius, uint32_t nq, float eps, const float *d_q_norm2, float max_norm, uint32_t dim, int l2,
                               float *d_thr, uint32_t *d_overflow, uint32_t *d_total, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    range_bound_kernel<<<(nq + 255) / 256, 256, 0, s>>>(d_radius, nq, eps, d_q_norm2, max_norm, dim, l2, d_thr, d_overflow, d_total);
    return cudaGetLastError();
}
cudaError_t launch_range_bound16(const void *d_queries, size_t qpitch, uint32_t nq, uint32_t dim, int dtype, const float *d_radius,
                                 float max_norm, float *d_thr, uint32_t *d_overflow, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    const uint8_t *qs = static_cast<const uint8_t *>(d_queries);
    if (dtype == DT_F16)
        range_bound16_kernel<DT_F16><<<(nq + 7) / 8, 256, 0, s>>>(qs, qpitch, nq, dim, d_radius, max_norm, d_thr, d_overflow);
    else if (dtype == DT_BF16)
        range_bound16_kernel<DT_BF16><<<(nq + 7) / 8, 256, 0, s>>>(qs, qpitch, nq, dim, d_radius, max_norm, d_thr, d_overflow);
    else
        return cudaErrorInvalidValue;
    return cudaGetLastError();
}
cudaError_t launch_range_refine(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t slots, uint64_t *d_cand,
                                const float *d_radius, const float *d_q_norm2, const float *d_thr, const uint32_t *d_overflow, uint64_t *d_out,
                                uint32_t *d_total, uint32_t *d_ok, uint32_t *d_cnt, uint32_t *d_off, cudaStream_t s, uint32_t cap) {
    if (nq == 0) return cudaSuccess;
    const uint8_t *rows = static_cast<const uint8_t *>(c.rows), *qs = static_cast<const uint8_t *>(d_queries);
    if (c.dtype == DT_F32 && c.metric == MT_L2)
        range_refine_kernel<DT_F32, MT_L2><<<nq, 256, 0, s>>>(rows, c.pitch, c.dim, qs, qpitch, slots, d_cand, d_radius, d_q_norm2, d_thr,
                                                              d_overflow, d_out, d_total, d_ok, d_cnt, d_off, cap);
    else if (c.dtype == DT_F32 && c.metric == MT_IP)
        range_refine_kernel<DT_F32, MT_IP><<<nq, 256, 0, s>>>(rows, c.pitch, c.dim, qs, qpitch, slots, d_cand, d_radius, d_q_norm2, d_thr,
                                                              d_overflow, d_out, d_total, d_ok, d_cnt, d_off, cap);
    else if (c.dtype == DT_F16 && c.metric == MT_IP) // the direct 16-bit route: inner product / cosine (normalised rows)
        range_refine_kernel<DT_F16, MT_IP><<<nq, 256, 0, s>>>(rows, c.pitch, c.dim, qs, qpitch, slots, d_cand, d_radius, d_q_norm2, d_thr,
                                                              d_overflow, d_out, d_total, d_ok, d_cnt, d_off, cap);
    else if (c.dtype == DT_BF16 && c.metric == MT_IP)
        range_refine_kernel<DT_BF16, MT_IP><<<nq, 256, 0, s>>>(rows, c.pitch, c.dim, qs, qpitch, slots, d_cand, d_radius, d_q_norm2, d_thr,
                                                               d_overflow, d_out, d_total, d_ok, d_cnt, d_off, cap);
    else
        return cudaErrorInvalidValue;
    return cudaGetLastError();
}
cudaError_t launch_range_pack(const uint64_t *d_cand, uint32_t nq, uint32_t slots, const uint32_t *d_overflow, uint32_t cap, uint64_t *d_out,
                              uint32_t *d_cnt, uint32_t *d_ok, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    range_pack_kernel<<<nq, 256, 0, s>>>(d_cand, slots, d_overflow, cap, d_out, d_cnt, d_ok);
    return cudaGetLastError();
}
cudaError_t launch_range_label_fold(const uint64_t *d_cand, uint32_t nq, uint32_t slots, const uint32_t *d_front, const uint32_t *d_overflow,
                                    const uint64_t *d_id_to_label, uint32_t cap, uint64_t *d_out, uint32_t *d_cnt, uint32_t *d_ok,
                                    uint32_t *d_flags, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    constexpr size_t smem = (size_t)kRangeFoldMaxHits * 12;
    cudaError_t e = cudaFuncSetAttribute(range_label_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    range_label_fold_kernel<<<nq, 512, smem, s>>>(d_cand, slots, d_front, d_overflow, d_id_to_label, cap, d_out, d_cnt, d_ok, d_flags);
    return cudaGetLastError();
}
cudaError_t launch_gather_queries(const void *d_src, size_t pitch, const float *d_src_n2, const uint32_t *d_idx, const uint32_t *d_count,
                                  uint32_t max_n, void *d_dst, float *d_dst_n2, cudaStream_t s) {
    if (max_n == 0) return cudaSuccess;
    gather_queries_kernel<<<std::min(max_n, 256u), 128, 0, s>>>(static_cast<const uint8_t *>(d_src), pitch, d_src_n2, d_idx, d_count,
                                                               static_cast<uint8_t *>(d_dst), d_dst_n2);
    return cudaGetLastError();
}

} // namespace rsb200
