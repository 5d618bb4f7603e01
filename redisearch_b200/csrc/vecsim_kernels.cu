// sm_90a kernels of the FLAT KNN path.  See DESIGN.md §3 for the roofline of each kernel.
//
//   scan_topk_kernel     fused distance scan + per-warp top-k lists   (HBM-bound: N*rowbytes)
//   final_select_kernel  candidates -> k smallest, sorted             (tiny)
//   scan_scores_kernel   all N distances of one query -> HBM          (HBM-bound; batch iterator,
//                                                                      range query, k > 128)
//   select_scores_kernel cursor-select over a score array             (N*4 bytes per pass)
//   range_compact_kernel scores <= radius -> compacted composites
//   gather_kernel        distances of listed rows (ad-hoc / hybrid)
//   gather_min_kernel    min fold over each listed label's rows (hybrid, multi-value index)
//   unpack / merge       reply formatting, G-way shard merge
//
// Replaces, on device: BruteForceIndex::topKQuery (VS/algorithms/brute_force/brute_force.h:243-291),
// rangeQuery (:293-326), BFS_BatchIterator::calculateScores (bfs_batch_iterator.h:24-40),
// BF_BatchIterator::getNextResults (bf_batch_iterator.h:176-200), getDistanceFrom_Unsafe
// (brute_force_single.h:200-212) and the distance functions of VS/spaces/.
#include "vecsim_kernels.h"
#include "distance_core.cuh"
#include "topk_common.cuh"

#include <algorithm>
#include <type_traits>
#include <mutex>

namespace rsb200 {

constexpr int kScanThreads = 256;
constexpr int kScanWarps = kScanThreads / 32;

int device_sm_count() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

// ------------------------------------------------------------------------------------------------
// per-warp list state in shared memory
// ------------------------------------------------------------------------------------------------
struct ListState {
    uint64_t *slots; // [k]
    uint64_t *worst; // [1]
    uint32_t *wpos;  // [1]
};

// All 32 lanes: finds the worst entry again after a slot changed.
__device__ __forceinline__ void list_rescan(const ListState &ls, uint32_t k, int lane) {
    uint64_t best = 0;
    uint32_t pos = 0;
    for (uint32_t p = lane; p < k; p += 32) {
        uint64_t v = ls.slots[p];
        if (v >= best) {
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
    if (lane == 0) {
        *ls.worst = best;
        *ls.wpos = pos;
    }
    __syncwarp();
}

// All 32 lanes; cand is warp-uniform.  Replaces the current worst entry, then rescans.
__device__ __forceinline__ void list_admit(const ListState &ls, uint32_t k, uint64_t cand, int lane) {
    if (lane == 0) ls.slots[*ls.wpos] = cand;
    __syncwarp();
    list_rescan(ls, k, lane);
}

// Label-aware list of a multi-value index (DESIGN.md §4.4): the list holds distinct labels, lab[p] = label of slots[p] (~0 for
// an empty slot), each at the best composite seen for it.  A candidate whose label is already listed replaces that entry only if
// it is smaller; a new label evicts the worst entry.  All 32 lanes; cand and label are warp-uniform, cand < *ls.worst.
__device__ __forceinline__ void list_admit_label(const ListState &ls, uint64_t *lab, uint32_t k, uint64_t cand, uint64_t label, int lane) {
    int hit = -1;
    for (uint32_t p0 = 0; p0 < k; p0 += 32) {
        const unsigned m = __ballot_sync(0xffffffffu, p0 + lane < k && lab[p0 + lane] == label);
        if (m) {
            hit = (int)(p0 + __ffs(m) - 1);
            break;
        }
    }
    if (hit >= 0) {
        const uint64_t cur = ls.slots[hit];
        __syncwarp();
        if (cand >= cur) return;
        if (lane == 0) ls.slots[hit] = cand;
        __syncwarp();
        list_rescan(ls, k, lane);
        return;
    }
    if (lane == 0) lab[*ls.wpos] = label;
    list_admit(ls, k, cand, lane);
}

// One CTA.  buf[0, n): composites in ascending order, kEmptySlot entries last (n <= 32 * blockDim.x).  Writes the first k
// composites whose label (id_to_label[row]) does not occur earlier in buf to out[0, k), kEmptySlot after them, and returns the
// number of distinct labels in buf to every thread.  Scratch in shared memory: lab [n], cnt [blockDim.x + 1].
__device__ uint32_t first_distinct_labels(const uint64_t *buf, uint32_t n, const uint64_t *__restrict__ id_to_label, uint32_t k,
                                          uint64_t *out, uint64_t *lab, uint32_t *cnt) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) lab[i] = buf[i] == kEmptySlot ? kEmptySlot : id_to_label[(uint32_t)buf[i]];
    __syncthreads();
    // each thread owns a contiguous chunk of positions: its first occurrences as a bit mask, then one exclusive scan of the counts
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x, i0 = min(n, threadIdx.x * per), i1 = min(n, i0 + per);
    uint32_t mine = 0;
    for (uint32_t i = i0; i < i1; i++) {
        if (buf[i] == kEmptySlot) break;
        const uint64_t l = lab[i];
        bool first = true;
        for (uint32_t j = 0; j < i && first; j++) first = lab[j] != l;
        if (first) mine |= 1u << (i - i0);
    }
    cnt[threadIdx.x] = __popc(mine);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (uint32_t t = 0; t < blockDim.x; t++) {
            const uint32_t c = cnt[t];
            cnt[t] = s;
            s += c;
        }
        cnt[blockDim.x] = s;
    }
    __syncthreads();
    uint32_t r = cnt[threadIdx.x];
    for (uint32_t i = i0; i < i1; i++)
        if ((mine >> (i - i0)) & 1u) {
            if (r < k) out[r] = buf[i];
            r++;
        }
    const uint32_t total = cnt[blockDim.x];
    for (uint32_t p = total + threadIdx.x; p < k; p += blockDim.x) out[p] = kEmptySlot;
    __syncthreads(); // lab / cnt may be reused
    return total;
}

// ------------------------------------------------------------------------------------------------
// fused scan + top-k
// ------------------------------------------------------------------------------------------------
struct ScanArgs {
    const uint8_t *rows;
    size_t pitch;
    uint32_t n_rows, dim;
    const uint8_t *queries; // device, 16B-aligned, qpitch (multiple of 16) apart
    size_t qpitch;
    uint32_t q_smem_pitch; // round16(query blob bytes)
    uint32_t nq, k, wq, lists_per_query;
    uint64_t *cand;
    const uint32_t *q_ok; // optional: queries already answered (coarse path verified) are skipped
    const uint32_t *abort; // optional (mapped host memory): non-zero = the caller has left (timeout), stop scanning
    uint32_t poll_mask;    // the flag is read every poll_mask + 1 tiles of a warp
    const uint64_t *id_to_label; // LAB: row -> label; the lists hold distinct labels (multi-value index)
};

// LAB: label-aware lists (list_admit_label), a label per slot in shared memory after the slots
template <int DT, int MT, int RT, int QT, bool QSMEM, bool LAB>
__global__ void __launch_bounds__(kScanThreads) scan_topk_kernel(const ScanArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    using Tile = DistTile<DT, MT, RT, QT>;
    using Map = typename Tile::Map;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t WQ = a.wq, WR = kScanWarps / WQ;
    const uint32_t qg = warp % WQ, rg = warp / WQ;
    const uint32_t q_cta0 = blockIdx.y * WQ * QT;
    const uint32_t q0 = q_cta0 + qg * QT;
    const uint32_t k = a.k;

    const size_t qs_bytes = QSMEM ? (size_t)WQ * QT * a.q_smem_pitch : 0;
    uint8_t *qs = smem;
    uint64_t *slots = reinterpret_cast<uint64_t *>(smem + qs_bytes);
    uint64_t *slab = slots + (size_t)kScanWarps * QT * k; // LAB only
    uint64_t *worst = slab + (LAB ? (size_t)kScanWarps * QT * k : 0);
    uint32_t *wpos = reinterpret_cast<uint32_t *>(worst + kScanWarps * QT);

    if (QSMEM) {
        const uint32_t vec_per_q = a.q_smem_pitch >> 4;
        const uint32_t total = WQ * QT * vec_per_q;
        for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
            const uint32_t qi = i / vec_per_q, vi = i - qi * vec_per_q;
            const uint32_t q = min(q_cta0 + qi, a.nq - 1);
            reinterpret_cast<uint4 *>(qs)[i] = reinterpret_cast<const uint4 *>(a.queries + (size_t)q * a.qpitch)[vi];
        }
    }
    {
        uint64_t *my = slots + (size_t)warp * QT * k;
        for (uint32_t p = lane; p < QT * k; p += 32) my[p] = kEmptySlot;
        if (LAB)
            for (uint32_t p = lane; p < QT * k; p += 32) slab[(size_t)warp * QT * k + p] = kEmptySlot;
        if (lane < QT) {
            worst[warp * QT + lane] = kEmptySlot;
            wpos[warp * QT + lane] = 0;
        }
    }
    __syncthreads();

    const uint8_t *qb[QT];
#pragma unroll
    for (int j = 0; j < QT; j++) {
        if (QSMEM)
            qb[j] = qs + (size_t)(qg * QT + j) * a.q_smem_pitch;
        else
            qb[j] = a.queries + (size_t)min(q0 + j, a.nq - 1) * a.qpitch;
    }

    const uint32_t ntiles = (a.n_rows + RT - 1) / RT;
    bool active = q0 < a.nq;
    if (active && a.q_ok) { // exact fallback of the tensor-core path: only unverified queries are scanned
        bool all_ok = true;
#pragma unroll
        for (int j = 0; j < QT; j++)
            if (q0 + j < a.nq && !a.q_ok[q0 + j]) all_ok = false;
        active = !all_ok;
    }
    if (active) {
        uint32_t since_poll = 0;
        for (uint32_t t = blockIdx.x * WR + rg; t < ntiles; t += gridDim.x * WR) {
            if (a.abort && (since_poll++ & a.poll_mask) == a.poll_mask) { // a host flag over PCIe: one lane reads it now and then
                uint32_t f = 0;
                if (lane == 0) f = *reinterpret_cast<const volatile uint32_t *>(a.abort);
                if (__shfl_sync(0xffffffffu, f, 0)) break; // the partial lists are published and then ignored by the host
            }
            const uint32_t r0 = t * RT;
            const uint8_t *rowb[RT];
#pragma unroll
            for (int i = 0; i < RT; i++) rowb[i] = a.rows + (size_t)min(r0 + i, a.n_rows - 1) * a.pitch;
            float d[Map::kPerLane];
            Tile::run(rowb, qb, a.dim, lane, d);
#pragma unroll
            for (int t2 = 0; t2 < Map::kPerLane; t2++) {
                const int idx = Map::value_index(lane, t2);
                const uint32_t row = r0 + idx / QT;
                const uint32_t j = idx % QT;
                const bool valid = Map::primary(lane) && row < a.n_rows && (q0 + j) < a.nq;
                const uint64_t comp = make_composite(d[t2], row);
                const uint64_t w = worst[warp * QT + j];
                unsigned pending = __ballot_sync(0xffffffffu, valid && comp < w);
                while (pending) {
                    const int src = __ffs(pending) - 1;
                    pending &= pending - 1;
                    const uint64_t c = shfl_u64(comp, src);
                    const uint32_t js = __shfl_sync(0xffffffffu, j, src);
                    ListState ls{slots + ((size_t)warp * QT + js) * k, worst + warp * QT + js, wpos + warp * QT + js};
                    if (LAB) {
                        if (c < *ls.worst) list_admit_label(ls, slab + ((size_t)warp * QT + js) * k, k, c, a.id_to_label[(uint32_t)c], lane);
                    } else if (c < *ls.worst) {
                        list_admit(ls, k, c, lane);
                    }
                }
            }
        }
    }
    __syncwarp();
    // publish this warp's lists
#pragma unroll
    for (int j = 0; j < QT; j++) {
        if (q0 + j < a.nq) {
            uint64_t *dst = a.cand + ((size_t)(q0 + j) * a.lists_per_query + blockIdx.x * WR + rg) * k;
            const uint64_t *src = slots + ((size_t)warp * QT + j) * k;
            for (uint32_t p = lane; p < k; p += 32) dst[p] = src[p];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// candidates -> k smallest per query, ascending
// ------------------------------------------------------------------------------------------------
// One CTA: the k smallest of src[0, m), ascending, into out[0, k).
__device__ __forceinline__ void final_select_cta(const uint64_t *__restrict__ src, uint32_t m, uint32_t k, uint64_t *__restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t sortn = next_pow2(kScanWarps * k);
    uint64_t *sortbuf = reinterpret_cast<uint64_t *>(smem); // [sortn]; first 8*k double as the lists
    uint64_t *worst = sortbuf + sortn;
    uint32_t *wpos = reinterpret_cast<uint32_t *>(worst + kScanWarps);

    for (uint32_t p = threadIdx.x; p < sortn; p += blockDim.x) sortbuf[p] = kEmptySlot;
    if (threadIdx.x < kScanWarps) {
        worst[threadIdx.x] = kEmptySlot;
        wpos[threadIdx.x] = 0;
    }
    __syncthreads();
    ListState ls{sortbuf + (size_t)warp * k, worst + warp, wpos + warp};
    for (uint32_t base = warp * 32; base < m; base += kScanThreads) {
        const uint32_t i = base + lane;
        const uint64_t c = (i < m) ? src[i] : kEmptySlot;
        unsigned pending = __ballot_sync(0xffffffffu, c < *ls.worst);
        while (pending) {
            const int s = __ffs(pending) - 1;
            pending &= pending - 1;
            const uint64_t cc = shfl_u64(c, s);
            if (cc < *ls.worst) list_admit(ls, k, cc, lane);
        }
    }
    bitonic_sort_smem(sortbuf, sortn);
    for (uint32_t p = threadIdx.x; p < k; p += blockDim.x) out[p] = sortbuf[p];
}

__global__ void __launch_bounds__(kScanThreads) final_select_kernel(const uint64_t *__restrict__ cand, uint32_t m,
                                                                    uint32_t k, uint64_t *__restrict__ out,
                                                                    const uint32_t *__restrict__ nq_dev) {
    if (nq_dev && blockIdx.x >= *nq_dev) return; // second tier: only the first *nq_dev positions hold lists
    final_select_cta(cand + (size_t)blockIdx.x * m, m, k, out + (size_t)blockIdx.x * k);
}

// The same over label-aware lists (multi-value index): each warp keeps the k best distinct labels of its share, and the first k
// distinct labels of the sorted union are the answer (per-list dedup, DESIGN.md §4.4).  out: (score, best row) composites.
__global__ void __launch_bounds__(kScanThreads) final_select_labels_kernel(const uint64_t *__restrict__ cand, uint32_t m, uint32_t k,
                                                                           const uint64_t *__restrict__ id_to_label,
                                                                           uint64_t *__restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t sortn = next_pow2(kScanWarps * k);
    uint64_t *sortbuf = reinterpret_cast<uint64_t *>(smem); // [sortn]; first 8*k double as the lists
    uint64_t *lab = sortbuf + sortn;                        // [sortn]: labels of the lists, then of the sorted entries
    uint64_t *worst = lab + sortn;
    uint32_t *wpos = reinterpret_cast<uint32_t *>(worst + kScanWarps);
    uint32_t *cnt = wpos + kScanWarps; // [kScanThreads + 1]
    const uint64_t *src = cand + (size_t)blockIdx.x * m;

    for (uint32_t p = threadIdx.x; p < sortn; p += blockDim.x) sortbuf[p] = lab[p] = kEmptySlot;
    if (threadIdx.x < kScanWarps) {
        worst[threadIdx.x] = kEmptySlot;
        wpos[threadIdx.x] = 0;
    }
    __syncthreads();
    ListState ls{sortbuf + (size_t)warp * k, worst + warp, wpos + warp};
    for (uint32_t base = warp * 32; base < m; base += kScanThreads) {
        const uint32_t i = base + lane;
        const uint64_t c = (i < m) ? src[i] : kEmptySlot;
        unsigned pending = __ballot_sync(0xffffffffu, c < *ls.worst);
        while (pending) {
            const int s = __ffs(pending) - 1;
            pending &= pending - 1;
            const uint64_t cc = shfl_u64(c, s);
            if (cc < *ls.worst) list_admit_label(ls, lab + (size_t)warp * k, k, cc, id_to_label[(uint32_t)cc], lane);
        }
    }
    bitonic_sort_smem(sortbuf, sortn);
    first_distinct_labels(sortbuf, sortn, id_to_label, k, out + (size_t)blockIdx.x * k, lab, cnt);
}

// Label stage after a row-level route (DESIGN.md §4.4), one CTA per query: rows[q] holds the query's K best rows, ascending.  The
// first kl distinct labels go to out[q] ([nq][kl], kEmptySlot after them).  The selection is proven iff the K rows hold at least
// kl distinct labels: lab_ok[q] = 1, flags[q] = the row stage's flag (row_ok[q], 1 without one); otherwise lab_ok[q] = 0 and
// flags[q] = 3 (the label-aware exact scan answers the query).
__global__ void __launch_bounds__(128) label_select_kernel(const uint64_t *__restrict__ rows, uint32_t K, const uint64_t *__restrict__ id_to_label,
                                                           uint32_t kl, const uint32_t *__restrict__ row_ok, uint64_t *__restrict__ out,
                                                           uint32_t *__restrict__ lab_ok, uint32_t *__restrict__ flags) {
    __shared__ uint64_t buf[kMaxFusedK], lab[kMaxFusedK];
    __shared__ uint32_t cnt[129];
    const uint32_t q = blockIdx.x;
    for (uint32_t i = threadIdx.x; i < K; i += blockDim.x) buf[i] = rows[(size_t)q * K + i];
    __syncthreads();
    const uint32_t distinct = first_distinct_labels(buf, K, id_to_label, kl, out + (size_t)q * kl, lab, cnt);
    if (threadIdx.x == 0) {
        const bool pass = distinct >= kl;
        lab_ok[q] = pass ? 1u : 0u;
        flags[q] = pass ? (row_ok ? row_ok[q] : 1u) : 3u;
    }
}

// ------------------------------------------------------------------------------------------------
// unfused: all scores of one query
// ------------------------------------------------------------------------------------------------
template <int DT, int MT>
__global__ void __launch_bounds__(kScanThreads) scan_scores_kernel(const uint8_t *rows, size_t pitch, uint32_t n_rows,
                                                                   uint32_t dim, const uint8_t *query,
                                                                   uint32_t q_smem_pitch, float *scores) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int RT = 4;
    using Tile = DistTile<DT, MT, RT, 1>;
    using Map = typename Tile::Map;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t i = threadIdx.x; i < (q_smem_pitch >> 4); i += blockDim.x)
        reinterpret_cast<uint4 *>(smem)[i] = reinterpret_cast<const uint4 *>(query)[i];
    __syncthreads();
    const uint8_t *qb[1] = {smem};
    const uint32_t ntiles = (n_rows + RT - 1) / RT;
    for (uint32_t t = blockIdx.x * kScanWarps + warp; t < ntiles; t += gridDim.x * kScanWarps) {
        const uint32_t r0 = t * RT;
        const uint8_t *rowb[RT];
#pragma unroll
        for (int i = 0; i < RT; i++) rowb[i] = rows + (size_t)min(r0 + i, n_rows - 1) * pitch;
        float d[Map::kPerLane];
        Tile::run(rowb, qb, dim, lane, d);
        const uint32_t row = r0 + Map::value_index(lane, 0);
        if (Map::primary(lane) && row < n_rows) scores[row] = d[0];
    }
}

// k smallest composites > cursor over a score array -> per-warp lists (part, warp) of cand; the array is shared by `parts` CTAs
__device__ __forceinline__ void select_scores_cta(const float *__restrict__ scores, uint32_t n, const uint64_t *__restrict__ cursor,
                                                  uint32_t k, uint64_t *__restrict__ cand, uint32_t part, uint32_t parts) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t *slots = reinterpret_cast<uint64_t *>(smem);
    uint64_t *worst = slots + (size_t)kScanWarps * k;
    uint32_t *wpos = reinterpret_cast<uint32_t *>(worst + kScanWarps);
    for (uint32_t p = threadIdx.x; p < kScanWarps * k; p += blockDim.x) slots[p] = kEmptySlot;
    if (threadIdx.x < kScanWarps) {
        worst[threadIdx.x] = kEmptySlot;
        wpos[threadIdx.x] = 0;
    }
    __syncthreads();
    const bool has_cursor = cursor != nullptr;
    const uint64_t lo = has_cursor ? *cursor : 0;
    ListState ls{slots + (size_t)warp * k, worst + warp, wpos + warp};
    const uint32_t gw = part * kScanWarps + warp, nw = parts * kScanWarps;
    for (uint64_t base = (uint64_t)gw * 32; base < n; base += (uint64_t)nw * 32) {
        const uint32_t i = (uint32_t)base + lane;
        bool valid = i < n;
        uint64_t c = kEmptySlot;
        if (valid) {
            c = make_composite(scores[i], i);
            valid = !has_cursor || c > lo;
        }
        unsigned pending = __ballot_sync(0xffffffffu, valid && c < *ls.worst);
        while (pending) {
            const int s = __ffs(pending) - 1;
            pending &= pending - 1;
            const uint64_t cc = shfl_u64(c, s);
            if (cc < *ls.worst) list_admit(ls, k, cc, lane);
        }
    }
    __syncwarp();
    uint64_t *dst = cand + (size_t)gw * k;
    for (uint32_t p = lane; p < k; p += 32) dst[p] = ls.slots[p];
}

__global__ void __launch_bounds__(kScanThreads) select_scores_kernel(const float *__restrict__ scores, uint32_t n,
                                                                     const uint64_t *__restrict__ cursor, uint32_t k,
                                                                     uint64_t *__restrict__ cand) {
    select_scores_cta(scores, n, cursor, k, cand, blockIdx.x, gridDim.x);
}

// ------------------------------------------------------------------------------------------------
// exact top-k of a batch for kMaxFusedK < k <= kMaxWideK (DESIGN.md §4.5): the unfused path of one query (all scores, then
// cursor selects of up to 128) with a query dimension.  The batch's positions are taken G at a time (a group); slot y of the
// group is position base + y, whose query is pos[base + y] (base + y without pos).  Only positions below *count (nq without
// count) are live: a CTA of a dead slot leaves at once, so a group whose positions are all answered reads nothing.
// ------------------------------------------------------------------------------------------------
struct WideGroup {
    const uint32_t *pos;   // nullable
    const uint32_t *count; // nullable
    uint32_t nq, base;
};
// live positions of the group from `base` on (0 = none)
__device__ __forceinline__ uint32_t wide_live(const WideGroup &g) {
    const uint32_t n = g.count ? min(*g.count, g.nq) : g.nq;
    return n > g.base ? n - g.base : 0u;
}
__device__ __forceinline__ uint32_t wide_query(const WideGroup &g, uint32_t slot) {
    return g.pos ? g.pos[g.base + slot] : g.base + slot;
}

struct WideScanArgs {
    const uint8_t *rows;
    size_t pitch;
    uint32_t n_rows, dim, wq, slots; // slots: positions in the group (scores holds slots x n_rows)
    const uint8_t *queries;
    size_t qpitch;
    WideGroup g;
    float *scores;
    const uint32_t *abort; // as ScanArgs
    uint32_t poll_mask;
};

// scores[slot][row] for the group's live slots: warp (qg, rg) of CTA y scores 8 slots against its row tiles (the arithmetic of
// scan_scores_kernel, which is that of the fused scan, query by query).  The wq query groups of a CTA share its rows through L1.
template <int DT, int MT>
__global__ void __launch_bounds__(kScanThreads) scan_scores_wide_kernel(const WideScanArgs a) {
    constexpr int RT = 4, QT = 8;
    using Tile = DistTile<DT, MT, RT, QT>;
    using Map = typename Tile::Map;
    const uint32_t live = min(wide_live(a.g), a.slots);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t WQ = a.wq, WR = kScanWarps / WQ, qg = warp % WQ, rg = warp / WQ;
    const uint32_t s0 = (blockIdx.y * WQ + qg) * QT;
    if (s0 >= live) return;
    const uint8_t *qb[QT];
#pragma unroll
    for (int j = 0; j < QT; j++) qb[j] = a.queries + (size_t)wide_query(a.g, min(s0 + j, live - 1)) * a.qpitch;
    const uint32_t ntiles = (a.n_rows + RT - 1) / RT;
    float *my_scores = a.scores + (size_t)s0 * a.n_rows;
    const uint32_t my_live = live - s0;
    uint32_t since_poll = 0;
    for (uint32_t t = blockIdx.x * WR + rg; t < ntiles; t += gridDim.x * WR) {
        if (a.abort && (since_poll++ & a.poll_mask) == a.poll_mask) {
            uint32_t f = 0;
            if (lane == 0) f = *reinterpret_cast<const volatile uint32_t *>(a.abort);
            if (__shfl_sync(0xffffffffu, f, 0)) break; // the caller has left: the scores are never read
        }
        const uint32_t r0 = t * RT;
        const uint8_t *rowb[RT];
#pragma unroll
        for (int i = 0; i < RT; i++) rowb[i] = a.rows + (size_t)min(r0 + i, a.n_rows - 1) * a.pitch;
        float d[Map::kPerLane];
        Tile::run(rowb, qb, a.dim, lane, d);
#pragma unroll
        for (int t2 = 0; t2 < Map::kPerLane; t2++) {
            const int idx = Map::value_index(lane, t2);
            const uint32_t row = r0 + idx / QT, j = idx % QT;
            if (Map::primary(lane) && row < a.n_rows && j < my_live) my_scores[(size_t)j * a.n_rows + row] = d[t2];
        }
    }
}

// chunk select of slot blockIdx.y: its scores, its cursor = the last composite of the previous chunk in its answer row
__global__ void __launch_bounds__(kScanThreads) select_scores_wide_kernel(const float *__restrict__ scores, uint32_t n, const WideGroup g,
                                                                          const uint64_t *__restrict__ out, uint32_t out_k, uint32_t first,
                                                                          uint32_t k, uint64_t *__restrict__ cand) {
    const uint32_t y = blockIdx.y;
    if (y >= wide_live(g)) return;
    const uint64_t *cursor = first ? out + (size_t)wide_query(g, y) * out_k + first - 1 : nullptr;
    select_scores_cta(scores + (size_t)y * n, n, cursor, k, cand + (size_t)y * gridDim.x * kScanWarps * k, blockIdx.x, gridDim.x);
}

// slot blockIdx.x: its lists -> its answer row, entries [first, first + k)
__global__ void __launch_bounds__(kScanThreads) final_select_wide_kernel(const uint64_t *__restrict__ cand, uint32_t m, const WideGroup g,
                                                                         uint64_t *__restrict__ out, uint32_t out_k, uint32_t first, uint32_t k) {
    const uint32_t y = blockIdx.x;
    if (y >= wide_live(g)) return;
    final_select_cta(cand + (size_t)y * m, m, k, out + (size_t)wide_query(g, y) * out_k + first);
}

__global__ void range_compact_kernel(const float *__restrict__ scores, uint32_t n, float radius,
                                     uint64_t *__restrict__ out, uint32_t *__restrict__ count) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float s = scores[i];
        if (s <= radius) { // brute_force.h:315 (NaN never passes)
            const uint32_t pos = atomicAdd(count, 1u);
            out[pos] = make_composite(s, i);
        }
    }
}

// exact range answers of a batch (DESIGN.md §4.11): slot blockIdx.y of the group, scores <= its query's radius into the query's
// cap slots (unordered), counted past cap
__global__ void __launch_bounds__(256) range_compact_wide_kernel(const float *__restrict__ scores, uint32_t n, const WideGroup g,
                                                                 const float *__restrict__ radii, uint32_t cap, uint64_t *__restrict__ out,
                                                                 uint32_t *__restrict__ counts) {
    const uint32_t y = blockIdx.y;
    if (y >= wide_live(g)) return;
    const uint32_t q = wide_query(g, y);
    const float r = radii[q];
    const float *mine = scores + (size_t)y * n;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float s = mine[i];
        if (s <= r) { // brute_force.h:315 (NaN never passes)
            const uint32_t pos = atomicAdd(counts + q, 1u);
            if (pos < cap) out[(size_t)q * cap + pos] = make_composite(s, i);
        }
    }
}

// exact range answers of a batch on a multi-value index (DESIGN.md §4.12), label-major over the CSR label table: slot blockIdx.y
// of the group, one thread per label, the smallest composite (score key, row) among the label's rows with score <= the radius;
// a label with such a row is appended to the query's cap slots (unordered) and counted past cap
__global__ void __launch_bounds__(256) range_label_wide_kernel(const float *__restrict__ scores, uint32_t n, const WideGroup g,
                                                               const float *__restrict__ radii, const uint32_t *__restrict__ label_off,
                                                               const uint32_t *__restrict__ label_rows, uint32_t n_labels, uint32_t cap,
                                                               uint64_t *__restrict__ out, uint32_t *__restrict__ counts) {
    const uint32_t y = blockIdx.y;
    if (y >= wide_live(g)) return;
    const uint32_t q = wide_query(g, y);
    const float r = radii[q];
    const float *mine = scores + (size_t)y * n;
    for (uint32_t l = blockIdx.x * blockDim.x + threadIdx.x; l < n_labels; l += gridDim.x * blockDim.x) {
        uint64_t best = ~0ull;
        for (uint32_t j = label_off[l], e = label_off[l + 1]; j < e; j++) {
            const uint32_t row = label_rows[j];
            const float s = mine[row];
            if (s <= r) { // brute_force.h:315 (NaN never passes)
                const uint64_t c = make_composite(s, row);
                best = c < best ? c : best;
            }
        }
        if (best != ~0ull) {
            const uint32_t pos = atomicAdd(counts + q, 1u);
            if (pos < cap) out[(size_t)q * cap + pos] = best;
        }
    }
}

// One CTA per query: its count and the composites (score key, row) in out[q][0, count) -> labels / scores in the reply order
// (finish_reply: BY_SCORE by (score, label), BY_ID by label), padded with -1 / NaN; a count past cap pads the whole row.  comp
// and labels are the same buffer: every composite is read before the first label is written.  Bitonic sort in shared memory
// over next_pow2(count) <= 4096 (key, label) pairs.
__global__ void __launch_bounds__(512) range_finish_kernel(int64_t *__restrict__ labels, float *__restrict__ scores,
                                                           const uint32_t *__restrict__ counts, uint32_t cap,
                                                           const uint64_t *__restrict__ id_to_label, int by_id) {
    extern __shared__ uint64_t s_lab[];
    const uint32_t q = blockIdx.x, cnt = counts[q];
    int64_t *L = labels + (size_t)q * cap;
    float *S = scores + (size_t)q * cap;
    const float nan = __int_as_float(0x7fffffff);
    if (cnt > cap || cnt == 0) {
        for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) L[i] = -1, S[i] = nan;
        return;
    }
    uint32_t n2 = 1;
    while (n2 < cnt) n2 <<= 1;
    uint32_t *s_key = reinterpret_cast<uint32_t *>(s_lab + n2);
    for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) {
        if (i < cnt) {
            const uint64_t c = (uint64_t)L[i];
            s_key[i] = (uint32_t)(c >> 32);
            s_lab[i] = id_to_label[(uint32_t)c];
        } else { // padding sorts last in either order
            s_key[i] = 0xFFFFFFFFu;
            s_lab[i] = ~0ull;
        }
    }
    __syncthreads();
    for (uint32_t k = 2; k <= n2; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) {
                const uint32_t p = i ^ j;
                if (p <= i) continue;
                const uint32_t ka = s_key[i], kb = s_key[p];
                const uint64_t la = s_lab[i], lb = s_lab[p];
                const bool b_first = by_id ? (lb < la || (lb == la && kb < ka)) : (kb < ka || (kb == ka && lb < la));
                if (b_first == ((i & k) == 0)) {
                    s_key[i] = kb, s_key[p] = ka;
                    s_lab[i] = lb, s_lab[p] = la;
                }
            }
            __syncthreads();
        }
    for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) {
        L[i] = i < cnt ? (int64_t)s_lab[i] : -1;
        S[i] = i < cnt ? key_to_float(s_key[i]) : nan;
    }
}

// ------------------------------------------------------------------------------------------------
// ad-hoc gather: one warp per listed row
// ------------------------------------------------------------------------------------------------
template <int DT, int MT>
__global__ void __launch_bounds__(kScanThreads) gather_kernel(const uint8_t *rows, size_t pitch, uint32_t dim,
                                                              const uint8_t *query, uint32_t q_smem_pitch,
                                                              const uint32_t *ids, uint32_t count, float *out) {
    extern __shared__ __align__(16) uint8_t smem[];
    using Tile = DistTile<DT, MT, 1, 1>;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t i = threadIdx.x; i < (q_smem_pitch >> 4); i += blockDim.x)
        reinterpret_cast<uint4 *>(smem)[i] = reinterpret_cast<const uint4 *>(query)[i];
    __syncthreads();
    const uint8_t *qb[1] = {smem};
    for (uint32_t w = blockIdx.x * kScanWarps + warp; w < count; w += gridDim.x * kScanWarps) {
        const uint32_t id = ids[w];
        if (id == 0xFFFFFFFFu) {
            if (lane == 0) out[w] = __uint_as_float(0x7FC00000u);
            continue;
        }
        const uint8_t *rowb[1] = {rows + (size_t)id * pitch};
        float d[1];
        Tile::run(rowb, qb, dim, lane, d);
        if (lane == 0) out[w] = d[0];
    }
}

// Ad-hoc gather of a multi-value index: one warp per listed label.  The label's rows are
// label_rows[offsets[l], offsets[l + 1]) in the order the host's label -> ids vector holds them; out[w] is
// getDistanceFrom_Unsafe's fold over them (brute_force_multi.h:224-241): dist = +inf, then
// dist = (dist < d) ? dist : d row by row.  Unlike fminf, a NaN row resets dist to NaN and the next
// row replaces it, so only a NaN in the LAST row survives.  Absent label (out of range or no rows) -> NaN.
template <int DT, int MT>
__global__ void __launch_bounds__(kScanThreads) gather_min_kernel(const uint8_t *rows, size_t pitch, uint32_t dim,
                                                                  const uint8_t *query, uint32_t q_smem_pitch,
                                                                  const uint32_t *labels, uint32_t count,
                                                                  const uint32_t *__restrict__ offsets, uint32_t n_labels,
                                                                  const uint32_t *__restrict__ label_rows, float *out) {
    extern __shared__ __align__(16) uint8_t smem[];
    using Tile = DistTile<DT, MT, 1, 1>;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t i = threadIdx.x; i < (q_smem_pitch >> 4); i += blockDim.x)
        reinterpret_cast<uint4 *>(smem)[i] = reinterpret_cast<const uint4 *>(query)[i];
    __syncthreads();
    const uint8_t *qb[1] = {smem};
    for (uint32_t w = blockIdx.x * kScanWarps + warp; w < count; w += gridDim.x * kScanWarps) {
        const uint32_t l = labels[w];
        uint32_t r = 0, e = 0;
        if (l < n_labels) {
            r = offsets[l];
            e = offsets[l + 1];
        }
        float dist = r < e ? __uint_as_float(0x7F800000u) : __uint_as_float(0x7FC00000u);
        uint32_t id = r < e ? label_rows[r] : 0u; // the next row id is loaded while this row is scored
#pragma unroll 1
        for (; r < e; r++) {
            const uint8_t *rowb[1] = {rows + (size_t)id * pitch};
            if (r + 1 < e) id = label_rows[r + 1];
            float d[1];
            Tile::run(rowb, qb, dim, lane, d);
            if (lane == 0) dist = (dist < d[0]) ? dist : d[0];
        }
        if (lane == 0) out[w] = dist;
    }
}

// ------------------------------------------------------------------------------------------------
// batched filtered KNN (DESIGN.md §4.6): nq filter lists of ragged lengths known only on the device.  Query q owns the flat score
// range [off[q], off[q + 1]) sized by its host cap; only its first min(*counts[q], cap) entries are live.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ragged_count(const RaggedBatch &b, uint32_t q) {
    const uint32_t cap = (uint32_t)(b.off[q + 1] - b.off[q]);
    const uint32_t *c = b.counts[q];
    return c ? min(*c, cap) : cap;
}

struct GatherRaggedArgs {
    const uint8_t *rows;
    size_t pitch;
    uint32_t dim;
    const uint8_t *queries;
    size_t qpitch;
    uint32_t q_smem_pitch;
    RaggedBatch b;
    const uint64_t *blk; // [nq + 1] first CTA of each query (prefix of ragged_blocks over the caps)
    uint64_t n_blocks;   // blk[nq]: chunks of kRaggedPerBlock entries; a grid of fewer CTAs strides over them
    const uint32_t *table; // single-value: docId -> row (0xFFFFFFFF absent); multi-value: CSR offsets [table_size + 1]
    uint32_t table_size;
    const uint32_t *label_rows; // multi-value: rows of each label in insertion order
    float *scores;
};
// the range form's (RANGE) outputs in place of the scores: radii [nq], the [nq][cap] composite slots and their counters (zeroed
// by the caller)
struct GatherRangeArgs : GatherRaggedArgs {
    const float *radii;
    uint32_t cap;
    uint64_t *out;
    uint32_t *counts;
};

// One chunk = kRaggedPerBlock consecutive entries of ONE query (its blob stays in shared memory), one warp per entry, with the
// arithmetic of gather_kernel (single-value) / gather_min_kernel's fold (multi-value).  A chunk past its query's device count ends
// after reading the count.  CTA i takes chunks i, i + gridDim.x, ... (one each when the grid covers them all).
// RANGE (DESIGN.md §4.13): no scores; an entry whose distance is <= its query's radius appends one composite (score key, row) to
// the query's cap slots, counted past cap.  Multi-value: the smallest composite over the label's PASSING rows (a NaN row never
// passes, so it cannot reset the fold as it does getDistanceFrom's).
template <int DT, int MT, bool MULTI, bool RANGE = false>
__global__ void __launch_bounds__(kScanThreads) gather_ragged_kernel(const std::conditional_t<RANGE, GatherRangeArgs, GatherRaggedArgs> a) {
    extern __shared__ __align__(16) uint8_t smem[];
    using Tile = DistTile<DT, MT, 1, 1>;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint64_t bid = blockIdx.x; bid < a.n_blocks; bid += gridDim.x) {
        uint32_t lo = 0, hi = a.b.nq; // blk[lo] <= bid < blk[hi]: lo is this chunk's query
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (a.blk[mid] <= bid) lo = mid;
            else hi = mid;
        }
        const uint32_t q = lo;
        const uint32_t e0 = (uint32_t)(bid - a.blk[q]) * kRaggedPerBlock;
        const uint32_t n = ragged_count(a.b, q);
        if (e0 >= n) { // the query's later chunks are past its count too: on to this CTA's first chunk of the next query
            bid += (a.blk[q + 1] - bid - 1) / gridDim.x * gridDim.x;
            continue;
        }
        const uint32_t e1 = min(n, e0 + kRaggedPerBlock);
        __syncthreads(); // the previous chunk's reads of the query blob are done
        const uint8_t *query = a.queries + (size_t)q * a.qpitch;
        for (uint32_t i = threadIdx.x; i < (a.q_smem_pitch >> 4); i += blockDim.x)
            reinterpret_cast<uint4 *>(smem)[i] = reinterpret_cast<const uint4 *>(query)[i];
        __syncthreads();
        const uint8_t *qb[1] = {smem};
        const uint32_t *ids = a.b.doc_ids[q];
        float *out = a.scores + a.b.off[q];
        for (uint32_t w = e0 + warp; w < e1; w += kScanWarps) {
            const uint32_t l = ids[w];
            if constexpr (RANGE) {
                const float radius = a.radii[q];
                uint64_t best = ~0ull;
                if (MULTI) {
                    uint32_t r = 0, e = 0;
                    if (l < a.table_size) {
                        r = a.table[l];
                        e = a.table[l + 1];
                    }
                    uint32_t id = r < e ? a.label_rows[r] : 0u;
#pragma unroll 1
                    for (; r < e; r++) {
                        const uint32_t row = id;
                        const uint8_t *rowb[1] = {a.rows + (size_t)row * a.pitch};
                        if (r + 1 < e) id = a.label_rows[r + 1];
                        float d[1];
                        Tile::run(rowb, qb, a.dim, lane, d);
                        if (lane == 0 && d[0] <= radius) { // brute_force.h:315 (NaN never passes)
                            const uint64_t c = make_composite(d[0], row);
                            best = c < best ? c : best;
                        }
                    }
                } else {
                    const uint32_t id = l < a.table_size ? a.table[l] : 0xFFFFFFFFu;
                    if (id == 0xFFFFFFFFu) continue;
                    const uint8_t *rowb[1] = {a.rows + (size_t)id * a.pitch};
                    float d[1];
                    Tile::run(rowb, qb, a.dim, lane, d);
                    if (lane == 0 && d[0] <= radius) best = make_composite(d[0], id);
                }
                if (lane == 0 && best != ~0ull) {
                    const uint32_t pos = atomicAdd(a.counts + q, 1u);
                    if (pos < a.cap) a.out[(size_t)q * a.cap + pos] = best;
                }
            } else if (MULTI) {
                uint32_t r = 0, e = 0;
                if (l < a.table_size) {
                    r = a.table[l];
                    e = a.table[l + 1];
                }
                float dist = r < e ? __uint_as_float(0x7F800000u) : __uint_as_float(0x7FC00000u);
                uint32_t id = r < e ? a.label_rows[r] : 0u;
#pragma unroll 1
                for (; r < e; r++) {
                    const uint8_t *rowb[1] = {a.rows + (size_t)id * a.pitch};
                    if (r + 1 < e) id = a.label_rows[r + 1];
                    float d[1];
                    Tile::run(rowb, qb, a.dim, lane, d);
                    if (lane == 0) dist = (dist < d[0]) ? dist : d[0];
                }
                if (lane == 0) out[w] = dist;
            } else {
                const uint32_t id = l < a.table_size ? a.table[l] : 0xFFFFFFFFu;
                if (id == 0xFFFFFFFFu) {
                    if (lane == 0) out[w] = __uint_as_float(0x7FC00000u);
                    continue;
                }
                const uint8_t *rowb[1] = {a.rows + (size_t)id * a.pitch};
                float d[1];
                Tile::run(rowb, qb, a.dim, lane, d);
                if (lane == 0) out[w] = d[0];
            }
        }
    }
}

// chunk select of query blockIdx.x / parts over its live scores; cursor = the last composite of the previous chunk in its row
__global__ void __launch_bounds__(kScanThreads) select_scores_ragged_kernel(const RaggedBatch b, const float *__restrict__ scores,
                                                                            uint32_t parts, const uint64_t *__restrict__ out, uint32_t out_k,
                                                                            uint32_t first, uint32_t k, uint64_t *__restrict__ cand) {
    const uint32_t q = blockIdx.x / parts, part = blockIdx.x - q * parts;
    const uint64_t *cursor = first ? out + (size_t)q * out_k + first - 1 : nullptr;
    select_scores_cta(scores + b.off[q], ragged_count(b, q), cursor, k, cand + (size_t)q * parts * kScanWarps * k, part, parts);
}

// query blockIdx.x: its lists -> its answer row, entries [first, first + k)
__global__ void __launch_bounds__(kScanThreads) final_select_ragged_kernel(const uint64_t *__restrict__ cand, uint32_t m,
                                                                           uint64_t *__restrict__ out, uint32_t out_k, uint32_t first,
                                                                           uint32_t k) {
    final_select_cta(cand + (size_t)blockIdx.x * m, m, k, out + (size_t)blockIdx.x * out_k + first);
}

// [nq][k] composites (position in the filter, ascending) -> docId labels and distances; NaN distances and empty slots -> -1 / NaN.
// They sort after every real entry, so a row's real entries are a prefix: counts[q] = its length.
// Hybrid batches (d.ok != NULL): a query with d.ok[q] != 0 takes row d.pos[q] of d.comp instead, whose composites carry docIds.
__global__ void unpack_ragged_kernel(const RaggedBatch b, const uint64_t *__restrict__ comp, uint32_t k, int64_t *__restrict__ labels,
                                     float *__restrict__ scores, uint32_t *__restrict__ counts, const DenseRows d) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)b.nq * k) return;
    const uint32_t q = (uint32_t)(i / k), j = (uint32_t)(i - (size_t)q * k);
    const bool dense = d.ok && d.ok[q] != 0;
    const uint64_t *row = dense ? d.comp + (size_t)d.pos[q] * k : comp + (size_t)q * k;
    const uint64_t c = row[j];
    const bool real = c < ((uint64_t)kNaNKey << 32);
    if (real) {
        labels[i] = dense ? (int64_t)(uint32_t)c : (int64_t)b.doc_ids[q][(uint32_t)c];
        scores[i] = key_to_float((uint32_t)(c >> 32));
    } else {
        labels[i] = -1;
        scores[i] = __uint_as_float(0x7FC00000u);
    }
    if (counts) {
        const bool next_real = j + 1 < k && row[j + 1] < ((uint64_t)kNaNKey << 32);
        if (real && !next_real) counts[q] = j + 1;
        if (j == 0 && !real) counts[q] = 0;
    }
}

// Row-space filter bitmaps of the dense queries of a hybrid batch (DESIGN.md §4.10): query p of the dense subset (dense_q[p] of the
// batch) sets bit `row` of bm[p] for every live entry docId -> table[docId] of its list; absent and deleted docIds set nothing.
// `parts` CTAs per dense query stride over its live entries.  bm must be zero.
__global__ void __launch_bounds__(256) filter_bitmap_kernel(const RaggedBatch b, const uint32_t *__restrict__ dense_q, uint32_t parts,
                                                            const uint32_t *__restrict__ table, uint32_t table_size, uint32_t *__restrict__ bm,
                                                            uint32_t words) {
    const uint32_t p = blockIdx.x / parts, part = blockIdx.x - p * parts, q = dense_q[p];
    const uint32_t n = ragged_count(b, q);
    const uint32_t *ids = b.doc_ids[q];
    uint32_t *mine = bm + (size_t)p * words;
    for (uint32_t e = part * blockDim.x + threadIdx.x; e < n; e += parts * blockDim.x) {
        const uint32_t l = ids[e];
        const uint32_t row = l < table_size ? table[l] : 0xFFFFFFFFu;
        if (row != 0xFFFFFFFFu) atomicOr(mine + (row >> 5), 1u << (row & 31));
    }
}

// Which queries of a hybrid batch the gather still answers: ok[q] = dense_ok[pos[q]] for a dense query (pos[q] != ~0), else 0;
// live[q] = 0 for a proven query, else its live filter length, and live_ptr[q] = &live[q] (the counts of the gather's RaggedBatch)
__global__ void hybrid_open_kernel(const RaggedBatch b, const uint32_t *__restrict__ pos, const uint32_t *__restrict__ dense_ok,
                                   uint32_t *__restrict__ ok, uint32_t *__restrict__ live, const uint32_t **__restrict__ live_ptr) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= b.nq) return;
    const uint32_t f = pos[q] != 0xFFFFFFFFu ? dense_ok[pos[q]] : 0u;
    ok[q] = f;
    live[q] = f ? 0u : ragged_count(b, q);
    live_ptr[q] = live + q;
}

// ------------------------------------------------------------------------------------------------
// reply formatting and shard merge
// ------------------------------------------------------------------------------------------------
__global__ void unpack_results_kernel(const uint64_t *__restrict__ comp, uint32_t total,
                                      const uint64_t *__restrict__ id_to_label, int64_t *__restrict__ labels,
                                      float *__restrict__ scores) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const uint64_t c = comp[i];
    if (c == kEmptySlot) {
        labels[i] = -1;
        scores[i] = __uint_as_float(0x7FC00000u);
    } else {
        const uint32_t id = (uint32_t)c;
        labels[i] = id_to_label ? (int64_t)id_to_label[id] : (int64_t)id;
        scores[i] = key_to_float((uint32_t)(c >> 32));
    }
}

// One CTA per query, rank sort of G*k (score,label) pairs; empty entries have label < 0.
// Shard g's arrays start score_stride floats / label_stride int64s after shard g-1's ([G][nq][k] arrays: nq*k; the
// packed exchange buffer of the shard group: one block of labels + scores per shard).
__global__ void merge_shards_kernel(const float *__restrict__ scores, const int64_t *__restrict__ labels, uint32_t G,
                                    uint32_t nq, uint32_t k, size_t score_stride, size_t label_stride,
                                    float *__restrict__ out_scores, int64_t *__restrict__ out_labels) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t q = blockIdx.x, n = G * k;
    uint32_t *keys = reinterpret_cast<uint32_t *>(smem);
    int64_t *labs = reinterpret_cast<int64_t *>(smem + (((size_t)n * 4 + 15) & ~(size_t)15));
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t g = i / k, p = i - g * k;
        const size_t src = (size_t)q * k + p;
        const int64_t l = labels[(size_t)g * label_stride + src];
        labs[i] = l;
        keys[i] = (l < 0) ? 0xFFFFFFFFu : orderable_key(scores[(size_t)g * score_stride + src]);
    }
    for (uint32_t i = threadIdx.x; i < k; i += blockDim.x) {
        out_labels[(size_t)q * k + i] = -1;
        out_scores[(size_t)q * k + i] = __uint_as_float(0x7FC00000u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t ki = keys[i];
        const int64_t li = labs[i];
        if (li < 0) continue;
        uint32_t rank = 0;
        for (uint32_t j = 0; j < n; j++) {
            const uint32_t kj = keys[j];
            const int64_t lj = labs[j];
            if (lj < 0) continue;
            // (score, label) lexicographic — VS/utils/query_result_utils.h:19-23; index breaks
            // exact duplicates (the same label cannot live on two shards).
            if (kj < ki || (kj == ki && (lj < li || (lj == li && j < i)))) rank++;
        }
        if (rank < k) {
            out_labels[(size_t)q * k + rank] = li;
            out_scores[(size_t)q * k + rank] = key_to_float(ki);
        }
    }
}

// Counted exchange blocks (DESIGN.md §6.1): per rank [labels int64 x nq*w][scores float x nq*w][counts u32 x nq], block_bytes
// apart.  Entry (score key, label) of a BY_SCORE run or (label, score key) of a BY_ID run: the composite the local calls sort by.
struct ListEntry {
    uint32_t key;
    uint64_t label;
};
__device__ __forceinline__ bool list_before(const ListEntry &a, const ListEntry &b, int by_id) {
    return by_id ? (a.label < b.label || (a.label == b.label && a.key < b.key)) : (a.key < b.key || (a.key == b.key && a.label < b.label));
}
__device__ __forceinline__ ListEntry list_entry(const int64_t *labels, const float *scores, size_t i) {
    return ListEntry{orderable_key(scores[i]), (uint64_t)labels[i]};
}

// One CTA per (query, rank): each entry of the rank's sorted run finds its place in the merged row as its index in the run plus,
// for every other run, a lower bound of its key (ties go to the smaller rank), so the places of all runs are a permutation of
// [0, sum of run lengths): O(G m log m) per query.  Scores are copied bit for bit.  The rank-0 CTA writes the count and pads the
// row past the merged entries; a failed rank (count UINT32_MAX) or, for range rows, a total past w pads the whole row.
__global__ void __launch_bounds__(256) merge_lists_kernel(const uint8_t *__restrict__ blocks, size_t block_bytes, uint32_t G, uint32_t nq,
                                                          uint32_t w, int range, int by_id, int64_t *__restrict__ out_labels,
                                                          float *__restrict__ out_scores, uint32_t *__restrict__ out_counts) {
    const size_t nw = (size_t)nq * w;
    const float nan = range ? __int_as_float(0x7fffffff) : __uint_as_float(0x7FC00000u); // the pad of range_finish / unpack_ragged
    for (uint64_t u = blockIdx.x; u < (uint64_t)nq * G; u += gridDim.x) {
        const uint32_t q = (uint32_t)(u / G), g = (uint32_t)(u - (uint64_t)q * G);
        uint64_t total = 0, merged = 0;
        bool failed = false;
        for (uint32_t h = 0; h < G; h++) {
            const uint32_t c = reinterpret_cast<const uint32_t *>(blocks + (size_t)h * block_bytes + nw * 12)[q];
            failed |= c == 0xFFFFFFFFu;
            total += c;
            merged += min(c, w);
        }
        const bool blank = failed || (range && total > w);
        int64_t *L = out_labels + (size_t)q * w;
        float *S = out_scores + (size_t)q * w;
        if (g == 0) {
            if (threadIdx.x == 0)
                out_counts[q] = failed ? 0xFFFFFFFFu : range ? (uint32_t)min(total, (uint64_t)0xFFFFFFFFu) : (uint32_t)min(total, (uint64_t)w);
            const uint32_t from = blank ? 0u : (uint32_t)min(merged, (uint64_t)w);
            for (uint32_t i = from + threadIdx.x; i < w; i += blockDim.x) L[i] = -1, S[i] = nan;
        }
        if (blank) continue;
        const uint8_t *mine = blocks + (size_t)g * block_bytes;
        const uint32_t m = min(reinterpret_cast<const uint32_t *>(mine + nw * 12)[q], w);
        const int64_t *ml = reinterpret_cast<const int64_t *>(mine) + (size_t)q * w;
        const float *ms = reinterpret_cast<const float *>(mine + nw * 8) + (size_t)q * w;
        for (uint32_t p = threadIdx.x; p < m; p += blockDim.x) {
            const ListEntry e = list_entry(ml, ms, p);
            uint64_t pos = p;
            for (uint32_t h = 0; h < G && pos < w; h++) {
                if (h == g) continue;
                const uint8_t *other = blocks + (size_t)h * block_bytes;
                const int64_t *hl = reinterpret_cast<const int64_t *>(other) + (size_t)q * w;
                const float *hs = reinterpret_cast<const float *>(other + nw * 8) + (size_t)q * w;
                uint32_t lo = 0, hi = min(reinterpret_cast<const uint32_t *>(other + nw * 12)[q], w);
                while (lo < hi) { // entries of run h placed before e: key <= e's for h < g, key < e's for h > g
                    const uint32_t mid = (lo + hi) >> 1;
                    const ListEntry o = list_entry(hl, hs, mid);
                    if (h < g ? !list_before(e, o, by_id) : list_before(o, e, by_id))
                        lo = mid + 1;
                    else
                        hi = mid;
                }
                pos += lo;
            }
            if (pos < w) L[pos] = ml[p], S[pos] = ms[p];
        }
    }
}

// ================================================================================================
// host side: dispatch
// ================================================================================================
static inline uint32_t round16(uint32_t v) { return (v + 15u) & ~15u; }

static uint32_t query_blob_bytes(const CorpusView &c) {
    switch (c.dtype) {
    case DT_F32: return c.dim * 4;
    case DT_F16:
    case DT_BF16: return c.dim * 2;
    default: return c.dim + (c.metric == MT_COS ? 4 : 0);
    }
}

template <typename K>
static cudaError_t ensure_smem(K kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

template <typename K>
static int occupancy(K kernel, size_t smem) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, kScanThreads, smem) != cudaSuccess || nb < 1) nb = 1;
    return nb;
}

constexpr size_t kMaxQuerySmem = 96 * 1024; // beyond this the batched scan reads queries through L1

constexpr size_t kMaxScanSmem = 227 * 1024; // opt-in shared memory per CTA on sm_90

ScanPlan plan_scan_topk(const CorpusView &c, uint32_t nq, uint32_t k, bool labels) {
    ScanPlan p{};
    p.qt = (nq == 1) ? 1 : 8;
    p.labels = labels;
    uint32_t groups = (nq + p.qt - 1) / p.qt;
    p.wq = groups >= 8 ? 8 : groups >= 4 ? 4 : groups >= 2 ? 2 : 1;
    const uint32_t qsp = round16(query_blob_bytes(c));
    p.grid_y = (groups + p.wq - 1) / p.wq;
    const uint32_t wr = kScanWarps / p.wq;
    // label-aware lists (multi-value index) carry a 64-bit label per slot: at k = 128 and 8 queries per warp that is 64 KB more,
    // 226 KB with 96 KB of staged queries; queries that would not fit are read through L1
    const size_t lists = (size_t)kScanWarps * p.qt * k * (labels ? 16 : 8) + (size_t)kScanWarps * p.qt * 12;
    size_t qs = (size_t)p.wq * p.qt * qsp;
    if (qs > kMaxQuerySmem || qs + lists > kMaxScanSmem) qs = 0;
    p.q_smem = qs != 0;
    p.smem_bytes = qs + lists;
    // persistent grid: resident CTAs only, split evenly over the query slices
    const int sms = device_sm_count();
    const uint32_t rt = 4;
    const uint32_t ntiles = (c.n_rows + rt - 1) / rt;
    uint32_t want = (ntiles + wr - 1) / wr;
    uint32_t resident = (uint32_t)sms * 2u;
    if (labels) // as many CTAs as the shared memory of an SM holds (228 KB, 1 KB reserved per CTA): one at k = 128
        resident = (uint32_t)sms * (uint32_t)std::max<size_t>(1, std::min<size_t>(2, (228 * 1024) / (p.smem_bytes + 1024)));
    p.grid_x = std::max(1u, std::min(want, std::max(1u, resident / p.grid_y)));
    p.lists_per_query = p.grid_x * wr;
    p.cand_elems = (size_t)nq * p.lists_per_query * k;
    return p;
}

template <int DT, int MT, int RT, int QT, bool QSMEM, bool LAB>
static cudaError_t launch_scan_inst(const ScanArgs &a, const ScanPlan &plan, cudaStream_t s) {
    auto kern = scan_topk_kernel<DT, MT, RT, QT, QSMEM, LAB>;
    cudaError_t e = ensure_smem(kern, plan.smem_bytes);
    if (e != cudaSuccess) return e;
    kern<<<dim3(plan.grid_x, plan.grid_y), kScanThreads, plan.smem_bytes, s>>>(a);
    return cudaGetLastError();
}

template <int DT, int MT, bool LAB>
static cudaError_t launch_scan_dml(const ScanArgs &a, const ScanPlan &plan, cudaStream_t s) {
    if (plan.qt == 1) return launch_scan_inst<DT, MT, 4, 1, true, LAB>(a, plan, s);
    if (plan.q_smem) return launch_scan_inst<DT, MT, 4, 8, true, LAB>(a, plan, s);
    return launch_scan_inst<DT, MT, 4, 8, false, LAB>(a, plan, s);
}

template <int DT, int MT>
static cudaError_t launch_scan_dm(const ScanArgs &a, const ScanPlan &plan, cudaStream_t s) {
    return plan.labels ? launch_scan_dml<DT, MT, true>(a, plan, s) : launch_scan_dml<DT, MT, false>(a, plan, s);
}

#define RSB_DISPATCH_DM(dtype, metric, CALL)                                                         \
    switch (dtype) {                                                                                 \
    case DT_F32:                                                                                     \
        if ((metric) == MT_L2) { CALL(DT_F32, MT_L2); } else { CALL(DT_F32, MT_IP); }                \
        break;                                                                                       \
    case DT_F16:                                                                                     \
        if ((metric) == MT_L2) { CALL(DT_F16, MT_L2); } else { CALL(DT_F16, MT_IP); }                \
        break;                                                                                       \
    case DT_BF16:                                                                                    \
        if ((metric) == MT_L2) { CALL(DT_BF16, MT_L2); } else { CALL(DT_BF16, MT_IP); }              \
        break;                                                                                       \
    case DT_I8:                                                                                      \
        if ((metric) == MT_L2) { CALL(DT_I8, MT_L2); }                                               \
        else if ((metric) == MT_IP) { CALL(DT_I8, MT_IP); }                                          \
        else { CALL(DT_I8, MT_COS); }                                                                \
        break;                                                                                       \
    case DT_U8:                                                                                      \
        if ((metric) == MT_L2) { CALL(DT_U8, MT_L2); }                                               \
        else if ((metric) == MT_IP) { CALL(DT_U8, MT_IP); }                                          \
        else { CALL(DT_U8, MT_COS); }                                                                \
        break;                                                                                       \
    }

__global__ void blend_kernel(const uint32_t *__restrict__ ok, const uint64_t *__restrict__ a, const uint64_t *__restrict__ b,
                             uint32_t total, uint32_t k, uint64_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) out[i] = ok[i / k] ? a[i] : b[i];
}
cudaError_t launch_blend(const uint32_t *d_ok, const uint64_t *d_a, const uint64_t *d_b, uint32_t nq, uint32_t k, uint64_t *d_out,
                         cudaStream_t s, LaunchCounters *ctr) {
    const uint32_t total = nq * k;
    if (!total) return cudaSuccess;
    blend_kernel<<<(total + 255) / 256, 256, 0, s>>>(d_ok, d_a, d_b, total, k, d_out);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_scan_topk(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t k,
                             const ScanPlan &plan, uint64_t *d_cand, cudaStream_t s, LaunchCounters *ctr,
                             const uint32_t *d_q_ok, const uint32_t *d_abort, const uint64_t *d_id_to_label) {
    if (nq == 0 || k == 0 || k > (uint32_t)kMaxFusedK || c.n_rows == 0) return cudaErrorInvalidValue;
    if (plan.labels != (d_id_to_label != nullptr)) return cudaErrorInvalidValue;
    ScanArgs a{};
    a.rows = static_cast<const uint8_t *>(c.rows);
    a.pitch = c.pitch;
    a.n_rows = c.n_rows;
    a.dim = c.dim;
    a.queries = static_cast<const uint8_t *>(d_queries);
    a.qpitch = qpitch;
    a.q_smem_pitch = round16(query_blob_bytes(c));
    a.nq = nq;
    a.k = k;
    a.wq = plan.wq;
    a.lists_per_query = plan.lists_per_query;
    a.cand = d_cand;
    a.q_ok = d_q_ok;
    a.abort = d_abort;
    a.poll_mask = nq >= 16 ? 15u : 255u; // a batched tile costs ~100x a single-query tile: keep the reaction time in milliseconds
    a.id_to_label = d_id_to_label;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_SCAN(DT, MT) e = launch_scan_dm<DT, MT>(a, plan, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_SCAN)
#undef CALL_SCAN
    if (ctr) ctr->launches++;
    return e;
}

cudaError_t launch_final_select(const uint64_t *d_cand, uint32_t nq, uint32_t m_per_query, uint32_t k,
                                uint64_t *d_out, cudaStream_t s, LaunchCounters *ctr, const uint32_t *d_nq_dev) {
    if (k == 0 || k > (uint32_t)kMaxFusedK) return cudaErrorInvalidValue;
    const size_t smem = (size_t)next_pow2(kScanWarps * k) * 8 + kScanWarps * 12;
    final_select_kernel<<<nq, kScanThreads, smem, s>>>(d_cand, m_per_query, k, d_out, d_nq_dev);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_final_select_labels(const uint64_t *d_cand, uint32_t nq, uint32_t m_per_query, uint32_t k, const uint64_t *d_id_to_label,
                                       uint64_t *d_out, cudaStream_t s, LaunchCounters *ctr) {
    if (k == 0 || k > (uint32_t)kMaxFusedK || !d_id_to_label) return cudaErrorInvalidValue;
    if (nq == 0) return cudaSuccess;
    const size_t smem = (size_t)next_pow2(kScanWarps * k) * 16 + kScanWarps * 12 + (kScanThreads + 1) * 4;
    cudaError_t e = ensure_smem(final_select_labels_kernel, smem);
    if (e != cudaSuccess) return e;
    final_select_labels_kernel<<<nq, kScanThreads, smem, s>>>(d_cand, m_per_query, k, d_id_to_label, d_out);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_label_select(const uint64_t *d_rows, uint32_t nq, uint32_t K, const uint64_t *d_id_to_label, uint32_t kl,
                                const uint32_t *d_row_ok, uint64_t *d_out, uint32_t *d_lab_ok, uint32_t *d_flags, cudaStream_t s,
                                LaunchCounters *ctr) {
    if (K == 0 || K > (uint32_t)kMaxFusedK || kl == 0 || kl > K || !d_id_to_label) return cudaErrorInvalidValue;
    if (nq == 0) return cudaSuccess;
    label_select_kernel<<<nq, 128, 0, s>>>(d_rows, K, d_id_to_label, kl, d_row_ok, d_out, d_lab_ok, d_flags);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

template <int DT, int MT>
static cudaError_t launch_scores_inst(const CorpusView &c, const void *d_query, float *d_scores, cudaStream_t s) {
    auto kern = scan_scores_kernel<DT, MT>;
    const uint32_t qsp = round16(query_blob_bytes(c));
    cudaError_t e = ensure_smem(kern, qsp);
    if (e != cudaSuccess) return e;
    const uint32_t ntiles = (c.n_rows + 3) / 4;
    const uint32_t want = (ntiles + kScanWarps - 1) / kScanWarps;
    const uint32_t grid = std::max(1u, std::min(want, (uint32_t)(device_sm_count() * occupancy(kern, qsp))));
    kern<<<grid, kScanThreads, qsp, s>>>(static_cast<const uint8_t *>(c.rows), c.pitch, c.n_rows, c.dim,
                                         static_cast<const uint8_t *>(d_query), qsp, d_scores);
    return cudaGetLastError();
}

cudaError_t launch_scan_scores(const CorpusView &c, const void *d_query, float *d_scores, cudaStream_t s,
                               LaunchCounters *ctr) {
    if (c.n_rows == 0) return cudaSuccess;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_SCORES(DT, MT) e = launch_scores_inst<DT, MT>(c, d_query, d_scores, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_SCORES)
#undef CALL_SCORES
    if (ctr) ctr->launches++;
    return e;
}

static uint32_t select_grid(uint32_t n) {
    const uint32_t want = (n + kScanThreads - 1) / kScanThreads;
    return std::max(1u, std::min(want, (uint32_t)device_sm_count() * 2u));
}
uint32_t plan_select_scores_lists(uint32_t n) { return select_grid(n) * kScanWarps; }

cudaError_t launch_select_scores(const float *d_scores, uint32_t n, const uint64_t *d_cursor, uint32_t k,
                                 uint64_t *d_cand, cudaStream_t s, LaunchCounters *ctr) {
    if (k == 0 || k > (uint32_t)kMaxFusedK) return cudaErrorInvalidValue;
    const size_t smem = (size_t)kScanWarps * k * 8 + kScanWarps * 12;
    select_scores_kernel<<<select_grid(n), kScanThreads, smem, s>>>(d_scores, n, d_cursor, k, d_cand);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

constexpr size_t kWideScoreBytes = size_t(1) << 30; // HBM for the scores of one group of the batched exact top-k

WidePlan plan_topk_wide(uint32_t n_rows, uint32_t nq) {
    WidePlan p{};
    const size_t n = std::max<uint32_t>(n_rows, 1);
    // at most 65,535 slots: the chunk select puts a group's slots on gridDim.y
    p.group = (uint32_t)std::max<size_t>(1, std::min<size_t>(std::min<size_t>(nq, 65535), kWideScoreBytes / (n * 4)));
    // the chunk selects of a group keep about two CTAs per SM busy in all: fewer lists per slot the more slots there are
    p.sel_grid = std::max(1u, std::min(select_grid(n_rows), (uint32_t)device_sm_count() * 2u / p.group));
    p.score_elems = (size_t)p.group * n_rows;
    p.cand_elems = (size_t)p.group * p.sel_grid * kScanWarps * kMaxFusedK;
    return p;
}

template <int DT, int MT>
static cudaError_t launch_scores_wide_inst(const WideScanArgs &a, cudaStream_t s) {
    auto kern = scan_scores_wide_kernel<DT, MT>;
    const uint32_t groups = (a.slots + 7) / 8, grid_y = (groups + a.wq - 1) / a.wq, wr = kScanWarps / a.wq;
    const uint32_t want = ((a.n_rows + 3) / 4 + wr - 1) / wr;
    const uint32_t resident = (uint32_t)(device_sm_count() * occupancy(kern, 0));
    const uint32_t grid_x = std::max(1u, std::min(want, std::max(1u, resident / grid_y)));
    kern<<<dim3(grid_x, grid_y), kScanThreads, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_topk_wide(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t k, const uint32_t *d_pos,
                             const uint32_t *d_count, const WidePlan &p, float *d_scores, uint64_t *d_cand, uint64_t *d_out,
                             const uint32_t *d_abort, cudaStream_t s, LaunchCounters *ctr) {
    if (k == 0 || k > (uint32_t)kMaxWideK || k > c.n_rows || p.group == 0) return cudaErrorInvalidValue;
    if (nq == 0) return cudaSuccess;
    WideScanArgs a{};
    a.rows = static_cast<const uint8_t *>(c.rows);
    a.pitch = c.pitch;
    a.n_rows = c.n_rows;
    a.dim = c.dim;
    a.queries = static_cast<const uint8_t *>(d_queries);
    a.qpitch = qpitch;
    a.scores = d_scores;
    a.abort = d_abort;
    a.poll_mask = 15u;
    const size_t fsmem = (size_t)next_pow2(kScanWarps * kMaxFusedK) * 8 + kScanWarps * 12;
    const size_t ssmem = (size_t)kScanWarps * kMaxFusedK * 8 + kScanWarps * 12;
    for (uint32_t base = 0; base < nq; base += p.group) {
        const WideGroup g{d_pos, d_count, nq, base};
        a.g = g;
        a.slots = std::min(p.group, nq - base);
        const uint32_t groups8 = (a.slots + 7) / 8;
        a.wq = groups8 >= 8 ? 8 : groups8 >= 4 ? 4 : groups8 >= 2 ? 2 : 1;
        cudaError_t e = cudaErrorInvalidValue;
#define CALL_SCORES_WIDE(DT, MT) e = launch_scores_wide_inst<DT, MT>(a, s)
        RSB_DISPATCH_DM(c.dtype, c.metric, CALL_SCORES_WIDE)
#undef CALL_SCORES_WIDE
        if (e != cudaSuccess) return e;
        if (ctr) ctr->launches++;
        for (uint32_t first = 0; first < k; first += kMaxFusedK) {
            const uint32_t chunk = std::min<uint32_t>(kMaxFusedK, k - first);
            select_scores_wide_kernel<<<dim3(p.sel_grid, a.slots), kScanThreads, ssmem, s>>>(d_scores, c.n_rows, g, d_out, k, first, chunk, d_cand);
            final_select_wide_kernel<<<a.slots, kScanThreads, fsmem, s>>>(d_cand, p.sel_grid * kScanWarps * chunk, g, d_out, k, first, chunk);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            if (ctr) ctr->launches += 2;
        }
    }
    return cudaSuccess;
}

cudaError_t launch_range_wide(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, const uint32_t *d_pos,
                              const uint32_t *d_count, const WidePlan &p, float *d_scores, const float *d_radii, uint32_t cap, uint64_t *d_out,
                              uint32_t *d_counts, const uint32_t *d_abort, cudaStream_t s, LaunchCounters *ctr, const uint32_t *label_off,
                              const uint32_t *label_rows, uint32_t n_labels) {
    if (cap == 0 || p.group == 0 || c.n_rows == 0) return cudaErrorInvalidValue;
    WideScanArgs a{};
    a.rows = static_cast<const uint8_t *>(c.rows);
    a.pitch = c.pitch;
    a.n_rows = c.n_rows;
    a.dim = c.dim;
    a.queries = static_cast<const uint8_t *>(d_queries);
    a.qpitch = qpitch;
    a.scores = d_scores;
    a.abort = d_abort;
    a.poll_mask = 15u;
    for (uint32_t base = 0; base < nq; base += p.group) {
        const WideGroup g{d_pos, d_count, nq, base};
        a.g = g;
        a.slots = std::min(p.group, nq - base);
        const uint32_t groups8 = (a.slots + 7) / 8;
        a.wq = groups8 >= 8 ? 8 : groups8 >= 4 ? 4 : groups8 >= 2 ? 2 : 1;
        cudaError_t e = cudaErrorInvalidValue;
#define CALL_SCORES_WIDE(DT, MT) e = launch_scores_wide_inst<DT, MT>(a, s)
        RSB_DISPATCH_DM(c.dtype, c.metric, CALL_SCORES_WIDE)
#undef CALL_SCORES_WIDE
        if (e != cudaSuccess) return e;
        const uint32_t items = label_off ? n_labels : c.n_rows;
        const uint32_t gx = std::max(1u, std::min((items + 255u) / 256u, (uint32_t)device_sm_count() * 8u / a.slots));
        if (label_off)
            range_label_wide_kernel<<<dim3(gx, a.slots), 256, 0, s>>>(d_scores, c.n_rows, g, d_radii, label_off, label_rows, n_labels, cap,
                                                                      d_out, d_counts);
        else
            range_compact_wide_kernel<<<dim3(gx, a.slots), 256, 0, s>>>(d_scores, c.n_rows, g, d_radii, cap, d_out, d_counts);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (ctr) ctr->launches += 2;
    }
    return cudaSuccess;
}

cudaError_t launch_range_finish(int64_t *d_labels, float *d_scores, const uint32_t *d_counts, uint32_t nq, uint32_t cap,
                                const uint64_t *d_id_to_label, bool by_id, cudaStream_t s, LaunchCounters *ctr) {
    if (nq == 0) return cudaSuccess;
    if (cap == 0 || cap > kRangeDeviceMaxCap) return cudaErrorInvalidValue;
    uint32_t n2 = 1;
    while (n2 < cap) n2 <<= 1;
    range_finish_kernel<<<nq, 512, (size_t)n2 * 12, s>>>(d_labels, d_scores, d_counts, cap, d_id_to_label, by_id ? 1 : 0);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_range_compact(const float *d_scores, uint32_t n, float radius, uint64_t *d_out, uint32_t *d_count,
                                 cudaStream_t s, LaunchCounters *ctr) {
    cudaError_t e = cudaMemsetAsync(d_count, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    if (n == 0) return cudaSuccess;
    const uint32_t grid = std::max(1u, std::min((n + 255u) / 256u, (uint32_t)device_sm_count() * 8u));
    range_compact_kernel<<<grid, 256, 0, s>>>(d_scores, n, radius, d_out, d_count);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

template <int DT, int MT>
static cudaError_t launch_gather_inst(const CorpusView &c, const void *d_query, const uint32_t *d_ids, uint32_t count,
                                      float *d_out, cudaStream_t s) {
    auto kern = gather_kernel<DT, MT>;
    const uint32_t qsp = round16(query_blob_bytes(c));
    cudaError_t e = ensure_smem(kern, qsp);
    if (e != cudaSuccess) return e;
    const uint32_t want = (count + kScanWarps - 1) / kScanWarps;
    const uint32_t grid = std::max(1u, std::min(want, (uint32_t)(device_sm_count() * occupancy(kern, qsp))));
    kern<<<grid, kScanThreads, qsp, s>>>(static_cast<const uint8_t *>(c.rows), c.pitch, c.dim,
                                         static_cast<const uint8_t *>(d_query), qsp, d_ids, count, d_out);
    return cudaGetLastError();
}

// labels (docIds) -> internal row ids through a dense device table; absent / out of range -> 0xFFFFFFFF (-> NaN distance)
__global__ void __launch_bounds__(256) map_labels_kernel(const uint32_t *__restrict__ labels, uint32_t n, const uint32_t *__restrict__ table,
                                                         uint32_t table_size, uint32_t *__restrict__ ids) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t l = labels[i];
        ids[i] = l < table_size ? table[l] : 0xFFFFFFFFu;
    }
}
cudaError_t launch_map_labels(const uint32_t *d_labels, uint32_t n, const uint32_t *d_table, uint32_t table_size, uint32_t *d_ids,
                              cudaStream_t s, LaunchCounters *ctr) {
    if (n == 0) return cudaSuccess;
    const uint32_t grid = std::min<uint32_t>((n + 255) / 256, (uint32_t)device_sm_count() * 8);
    map_labels_kernel<<<grid, 256, 0, s>>>(d_labels, n, d_table, table_size, d_ids);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}
// out_labels[i] = labels[index part of comp[i]] (0 for empty slots)
__global__ void pick_labels_kernel(const uint64_t *__restrict__ comp, uint32_t k, const uint32_t *__restrict__ labels, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k) out[i] = comp[i] == kEmptySlot ? 0u : labels[(uint32_t)comp[i]];
}
cudaError_t launch_pick_labels(const uint64_t *d_comp, uint32_t k, const uint32_t *d_labels, uint32_t *d_out, cudaStream_t s,
                               LaunchCounters *ctr) {
    if (k == 0) return cudaSuccess;
    pick_labels_kernel<<<(k + 127) / 128, 128, 0, s>>>(d_comp, k, d_labels, d_out);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_gather_distances(const CorpusView &c, const void *d_query, const uint32_t *d_ids, uint32_t count,
                                    float *d_out, cudaStream_t s, LaunchCounters *ctr) {
    if (count == 0) return cudaSuccess;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_GATHER(DT, MT) e = launch_gather_inst<DT, MT>(c, d_query, d_ids, count, d_out, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_GATHER)
#undef CALL_GATHER
    if (ctr) ctr->launches++;
    return e;
}

template <int DT, int MT>
static cudaError_t launch_gather_min_inst(const CorpusView &c, const void *d_query, const uint32_t *d_labels, uint32_t count,
                                          const uint32_t *d_offsets, uint32_t n_labels, const uint32_t *d_label_rows, float *d_out,
                                          cudaStream_t s) {
    auto kern = gather_min_kernel<DT, MT>;
    const uint32_t qsp = round16(query_blob_bytes(c));
    cudaError_t e = ensure_smem(kern, qsp);
    if (e != cudaSuccess) return e;
    const uint32_t want = (count + kScanWarps - 1) / kScanWarps;
    const uint32_t grid = std::max(1u, std::min(want, (uint32_t)(device_sm_count() * occupancy(kern, qsp))));
    kern<<<grid, kScanThreads, qsp, s>>>(static_cast<const uint8_t *>(c.rows), c.pitch, c.dim, static_cast<const uint8_t *>(d_query), qsp,
                                         d_labels, count, d_offsets, n_labels, d_label_rows, d_out);
    return cudaGetLastError();
}

cudaError_t launch_gather_min_distances(const CorpusView &c, const void *d_query, const uint32_t *d_labels, uint32_t count,
                                        const uint32_t *d_offsets, uint32_t n_labels, const uint32_t *d_label_rows, float *d_out,
                                        cudaStream_t s, LaunchCounters *ctr) {
    if (count == 0) return cudaSuccess;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_GATHER_MIN(DT, MT) e = launch_gather_min_inst<DT, MT>(c, d_query, d_labels, count, d_offsets, n_labels, d_label_rows, d_out, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_GATHER_MIN)
#undef CALL_GATHER_MIN
    if (ctr) ctr->launches++;
    return e;
}

template <int DT, int MT, bool MULTI, bool RANGE = false, class Args>
static cudaError_t launch_gather_ragged_inst(const Args &a, uint64_t grid, cudaStream_t s) {
    auto kern = gather_ragged_kernel<DT, MT, MULTI, RANGE>;
    cudaError_t e = ensure_smem(kern, a.q_smem_pitch);
    if (e != cudaSuccess) return e;
    kern<<<(uint32_t)grid, kScanThreads, a.q_smem_pitch, s>>>(a);
    return cudaGetLastError();
}

static GatherRaggedArgs gather_ragged_args(const CorpusView &c, const void *d_queries, size_t qpitch, const RaggedBatch &b, const uint64_t *d_blk,
                                           uint64_t n_blocks, const uint32_t *d_table, uint32_t table_size, const uint32_t *d_label_rows) {
    GatherRaggedArgs a{};
    a.rows = static_cast<const uint8_t *>(c.rows);
    a.pitch = c.pitch;
    a.dim = c.dim;
    a.queries = static_cast<const uint8_t *>(d_queries);
    a.qpitch = qpitch;
    a.q_smem_pitch = round16(query_blob_bytes(c));
    a.b = b;
    a.blk = d_blk;
    a.n_blocks = n_blocks;
    a.table = d_table;
    a.table_size = table_size;
    a.label_rows = d_label_rows;
    return a;
}

cudaError_t launch_gather_ragged(const CorpusView &c, const void *d_queries, size_t qpitch, const RaggedBatch &b, const uint64_t *d_blk,
                                 uint64_t n_blocks, const uint32_t *d_table, uint32_t table_size, const uint32_t *d_label_rows, float *d_scores,
                                 cudaStream_t s, LaunchCounters *ctr, uint64_t max_grid) {
    if (n_blocks == 0 || b.nq == 0) return cudaSuccess;
    const uint64_t grid = max_grid ? std::min(n_blocks, max_grid) : n_blocks;
    if (grid > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    GatherRaggedArgs a = gather_ragged_args(c, d_queries, qpitch, b, d_blk, n_blocks, d_table, table_size, d_label_rows);
    a.scores = d_scores;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_GATHER_RAGGED(DT, MT)                                                                       \
    e = d_label_rows ? launch_gather_ragged_inst<DT, MT, true>(a, grid, s) : launch_gather_ragged_inst<DT, MT, false>(a, grid, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_GATHER_RAGGED)
#undef CALL_GATHER_RAGGED
    if (ctr) ctr->launches++;
    return e;
}

cudaError_t launch_gather_ragged_range(const CorpusView &c, const void *d_queries, size_t qpitch, const RaggedBatch &b, const uint64_t *d_blk,
                                       uint64_t n_blocks, const uint32_t *d_table, uint32_t table_size, const uint32_t *d_label_rows,
                                       const float *d_radii, uint32_t cap, uint64_t *d_out, uint32_t *d_counts, cudaStream_t s, LaunchCounters *ctr,
                                       uint64_t max_grid) {
    if (n_blocks == 0 || b.nq == 0) return cudaSuccess;
    const uint64_t grid = max_grid ? std::min(n_blocks, max_grid) : n_blocks;
    if (grid > 0x7FFFFFFFull || cap == 0) return cudaErrorInvalidValue;
    GatherRangeArgs a;
    static_cast<GatherRaggedArgs &>(a) = gather_ragged_args(c, d_queries, qpitch, b, d_blk, n_blocks, d_table, table_size, d_label_rows);
    a.radii = d_radii;
    a.cap = cap;
    a.out = d_out;
    a.counts = d_counts;
    cudaError_t e = cudaErrorInvalidValue;
#define CALL_GATHER_RANGE(DT, MT)                                                                        \
    e = d_label_rows ? launch_gather_ragged_inst<DT, MT, true, true>(a, grid, s) : launch_gather_ragged_inst<DT, MT, false, true>(a, grid, s)
    RSB_DISPATCH_DM(c.dtype, c.metric, CALL_GATHER_RANGE)
#undef CALL_GATHER_RANGE
    if (ctr) ctr->launches++;
    return e;
}

uint32_t plan_ragged_select_parts(size_t max_cap, uint32_t nq) {
    // about two CTAs per SM over the whole batch, never more CTAs for a query than its largest list can feed
    const uint32_t budget = std::max(1u, (uint32_t)device_sm_count() * 2u / std::max(1u, nq));
    return std::max(1u, std::min(select_grid((uint32_t)std::min<size_t>(max_cap, 0xFFFFFFFFu)), budget));
}

cudaError_t launch_topk_ragged(const RaggedBatch &b, const float *d_scores, uint32_t k, uint32_t parts, uint64_t *d_cand, uint64_t *d_out,
                               cudaStream_t s, LaunchCounters *ctr) {
    if (k == 0 || k > (uint32_t)kMaxWideK || parts == 0) return cudaErrorInvalidValue;
    if (b.nq == 0) return cudaSuccess;
    const uint64_t sel_ctas = (uint64_t)b.nq * parts;
    if (sel_ctas > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    for (uint32_t first = 0; first < k; first += kMaxFusedK) {
        const uint32_t chunk = std::min<uint32_t>(kMaxFusedK, k - first);
        const size_t ssmem = (size_t)kScanWarps * chunk * 8 + kScanWarps * 12;
        const size_t fsmem = (size_t)next_pow2(kScanWarps * chunk) * 8 + kScanWarps * 12;
        select_scores_ragged_kernel<<<(uint32_t)sel_ctas, kScanThreads, ssmem, s>>>(b, d_scores, parts, d_out, k, first, chunk, d_cand);
        final_select_ragged_kernel<<<b.nq, kScanThreads, fsmem, s>>>(d_cand, parts * kScanWarps * chunk, d_out, k, first, chunk);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        if (ctr) ctr->launches += 2;
    }
    return cudaSuccess;
}

cudaError_t launch_unpack_ragged(const RaggedBatch &b, const uint64_t *d_comp, uint32_t k, int64_t *d_labels, float *d_scores,
                                 uint32_t *d_counts, cudaStream_t s, LaunchCounters *ctr, const DenseRows &dense) {
    const size_t total = (size_t)b.nq * k;
    if (total == 0) return cudaSuccess;
    if ((total + 255) / 256 > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    unpack_ragged_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(b, d_comp, k, d_labels, d_scores, d_counts, dense);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_filter_bitmaps(const RaggedBatch &b, const uint32_t *d_dense_q, uint32_t n_dense, size_t max_cap, const uint32_t *d_table,
                                  uint32_t table_size, uint32_t *d_bm, uint32_t words, cudaStream_t s, LaunchCounters *ctr) {
    if (n_dense == 0) return cudaSuccess;
    // about four CTAs per SM over the dense queries, never more per query than its largest list can feed
    const uint32_t parts = (uint32_t)std::max<size_t>(1, std::min<size_t>((max_cap + 255) / 256,
                                                                           std::max(1u, (uint32_t)device_sm_count() * 4u / n_dense)));
    if ((uint64_t)n_dense * parts > 0x7FFFFFFFull) return cudaErrorInvalidValue;
    filter_bitmap_kernel<<<n_dense * parts, 256, 0, s>>>(b, d_dense_q, parts, d_table, table_size, d_bm, words);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_hybrid_open(const RaggedBatch &b, const uint32_t *d_pos, const uint32_t *d_dense_ok, uint32_t *d_ok, uint32_t *d_live,
                               const uint32_t **d_live_ptr, cudaStream_t s, LaunchCounters *ctr) {
    if (b.nq == 0) return cudaSuccess;
    hybrid_open_kernel<<<(b.nq + 255) / 256, 256, 0, s>>>(b, d_pos, d_dense_ok, d_ok, d_live, d_live_ptr);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_unpack_results(const uint64_t *d_comp, uint32_t nq, uint32_t k, const uint64_t *d_id_to_label,
                                  int64_t *d_labels, float *d_scores, cudaStream_t s, LaunchCounters *ctr) {
    const uint32_t total = nq * k;
    if (total == 0) return cudaSuccess;
    unpack_results_kernel<<<(total + 255) / 256, 256, 0, s>>>(d_comp, total, d_id_to_label, d_labels, d_scores);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_merge_shards(const float *d_scores, const int64_t *d_labels, uint32_t G, uint32_t nq, uint32_t k,
                                float *d_out_scores, int64_t *d_out_labels, cudaStream_t s, LaunchCounters *ctr,
                                size_t score_stride, size_t label_stride) {
    if (score_stride == 0) score_stride = (size_t)nq * k;
    if (label_stride == 0) label_stride = (size_t)nq * k;
    if (nq == 0 || k == 0 || G == 0) return cudaSuccess;
    const size_t n = (size_t)G * k;
    const size_t smem = ((n * 4 + 15) & ~(size_t)15) + n * 8;
    if (smem > 200 * 1024) return cudaErrorInvalidValue;
    cudaError_t e = ensure_smem(merge_shards_kernel, smem);
    if (e != cudaSuccess) return e;
    merge_shards_kernel<<<nq, 256, smem, s>>>(d_scores, d_labels, G, nq, k, score_stride, label_stride, d_out_scores, d_out_labels);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

cudaError_t launch_merge_lists(const void *d_blocks, size_t block_bytes, uint32_t G, uint32_t nq, uint32_t w, bool range, bool by_id,
                               int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s, LaunchCounters *ctr) {
    if (nq == 0) return cudaSuccess;
    const uint64_t grid = std::min<uint64_t>((uint64_t)nq * G, 1u << 20);
    merge_lists_kernel<<<(unsigned)grid, 256, 0, s>>>(static_cast<const uint8_t *>(d_blocks), block_bytes, G, nq, w, range ? 1 : 0,
                                                      by_id ? 1 : 0, d_out_labels, d_out_scores, d_out_counts);
    if (ctr) ctr->launches++;
    return cudaGetLastError();
}

} // namespace rsb200
