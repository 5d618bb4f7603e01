// sm_90a kernels of the posting-list path (HBM-bound integer work: no tensor cores here).
//
//   decode_blocks_kernel   IndexBlock bytes -> (docId, freq) arrays, one thread per block
//   intersect_kernel       k-way AND: the shortest list is cut into 1024-entry chunks (one CTA each);
//                          for every other list the CTA gallops to the chunk's docId window with two
//                          binary searches, stages the window in shared memory (coalesced) and
//                          resolves membership there; survivors are compacted in order
//   scan_kernel            exclusive prefix sum of per-chunk counts (single CTA)
//   gather_score_kernel    survivors -> ascending docIds + per-child freqs + score
//   union: mark / popc / expand / fill kernels over a docId bitmap (order-preserving, O(sum |L|))
//   ub_*: the same for a whole batch of ORs / numeric range filters, ragged over every list of every query
//   ifb_*: the AND probe of intersect_kernel for a whole batch of filter-mode ANDs, ragged over every query's driver chunks
//   score_kernel           the reference's scorers, expression tree by expression tree
//   topn_kernel            (score desc, docId asc) selection
//
// Replaces on device: Intersection::read / find_consensus (RS/rqe_iterators/src/intersection.rs:245-452),
// UnionFlat::read_full (union_flat.rs:324-348), IndexReader::next_record + codecs
// (RS/inverted_index/src/reader/core.rs:245-277, codec/*.rs), the default scorers
// (src/ext/default.c:68-461) and RPSorter's ranking (src/result_processor.c:752-850).
#include "ii_kernels.h"
#include "ii_codec.h"
#include "topk_common.cuh"

#include <algorithm>

namespace rsb200 {

// ------------------------------------------------------------------------------------------------
// device decode: one thread per IndexBlock; the record layouts live in ii_codec.h (shared with the host decoder)
// ------------------------------------------------------------------------------------------------
// What lands in out_masks: the record's 32-bit field mask, or — for the u128 masks of the *Wide codecs — whether it meets the
// 128-bit filter (1 / 0), so that the ordered compaction downstream stays a 32-bit `mask & filter` test (filter 1).
__device__ __forceinline__ uint32_t mask_word(const IIRecord &r, int codec, uint64_t wf_lo, uint64_t wf_hi) {
    if (!ii_codec_is_wide(codec)) return (uint32_t)r.mask_lo;
    return ((r.mask_lo & wf_lo) | (r.mask_hi & wf_hi)) != 0 ? 1u : 0u;
}

__global__ void decode_blocks_kernel(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ byte_off,
                                     const uint64_t *__restrict__ first_id, const uint32_t *__restrict__ entry_off,
                                     uint32_t nblocks, int codec, uint64_t wf_lo, uint64_t wf_hi, uint32_t *__restrict__ out_ids,
                                     uint32_t *__restrict__ out_freqs, uint32_t *__restrict__ out_masks) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const uint8_t *p = bytes + byte_off[b];
    const uint32_t n = entry_off[b + 1] - entry_off[b];
    uint32_t o = entry_off[b];
    const uint64_t base0 = first_id[b];
    uint64_t last = base0; // reader resets the delta base to first_doc_id on block entry (reader/core.rs:430-440)
    for (uint32_t e = 0; e < n; e++, o++) {
        IIRecord r;
        p = ii_decode_record<false>(p, nullptr, codec, r);
        const uint64_t id = (codec == 5 ? base0 : last) + r.delta; // raw doc ids: delta from the block's first id
        last = id;
        out_ids[o] = (uint32_t)id;
        out_freqs[o] = r.freq;
        if (out_masks) out_masks[o] = mask_word(r, codec, wf_lo, wf_hi);
    }
}

// The same, for a whole batch of posting lists at once, with the block bytes staged in shared memory: a CTA of 128 threads
// owns 128 consecutive blocks of the gathered byte stream (contiguous in HBM), copies their bytes into shared memory with
// coalesced 16-byte loads and then every thread walks its own block there — the qint / varint records of a block are a
// dependent chain (the lead byte of record e+1 is only known after record e), so the parallelism is across blocks, and
// what the one-thread-per-block kernel above loses is byte-granular global loads.  Tables are 32-bit (a batch is < 4 GB).
// out_masks may be NULL.  Blocks whose bytes do not fit the staging area are read from global memory.
constexpr int kDecodeThreads = 128;
constexpr uint32_t kDecodeSmem = 96 * 1024;
__global__ void __launch_bounds__(kDecodeThreads) decode_blocks_staged_kernel(const uint8_t *__restrict__ bytes, const uint32_t *__restrict__ byte_off,
                                                                              const uint32_t *__restrict__ first_id,
                                                                              const uint32_t *__restrict__ entry_off, uint32_t nblocks, int codec,
                                                                              uint32_t *__restrict__ out_ids, uint32_t *__restrict__ out_freqs,
                                                                              uint32_t *__restrict__ out_masks, uint32_t *__restrict__ out_off_pos,
                                                                              uint32_t *__restrict__ out_off_len) {
    extern __shared__ __align__(16) uint8_t s_bytes[];
    const uint32_t b0 = blockIdx.x * kDecodeThreads;
    const uint32_t b1 = min(b0 + (uint32_t)kDecodeThreads, nblocks);
    const uint32_t lo = byte_off[b0] & ~15u, hi = byte_off[b1]; // 16-byte aligned start: the gathered stream is 16-byte aligned
    const bool staged = hi - lo <= kDecodeSmem;
    if (staged) {
        const uint4 *src = reinterpret_cast<const uint4 *>(bytes + lo);
        uint4 *dst = reinterpret_cast<uint4 *>(s_bytes);
        const uint32_t n16 = (hi - lo + 15) / 16;
        for (uint32_t t = threadIdx.x; t < n16; t += kDecodeThreads) dst[t] = src[t]; // the stream is padded to 16 bytes
        __syncthreads();
    }
    const uint32_t b = b0 + threadIdx.x;
    if (b >= b1) return;
    const uint8_t *p = staged ? s_bytes + (byte_off[b] - lo) : bytes + byte_off[b];
    const uint8_t *const p0 = p; // position of a byte in the gathered stream = byte_off[b] + (its address - p0)
    const uint32_t stream0 = byte_off[b];
    const uint32_t n = entry_off[b + 1] - entry_off[b];
    uint32_t o = entry_off[b];
    const uint32_t base0 = first_id[b];
    uint32_t last = base0; // the reader resets the delta base to first_doc_id on block entry (reader/core.rs:430-440)
    for (uint32_t e = 0; e < n; e++, o++) {
        IIRecord r;
        p = ii_decode_record<false>(p, nullptr, codec, r);
        const uint32_t id = (codec == 5 ? base0 : last) + (uint32_t)r.delta;
        if (out_off_pos) { // the term's position bytes stay where they are, in the gathered stream kept on the device
            out_off_pos[o] = stream0 + (uint32_t)(r.offsets - p0);
            out_off_len[o] = r.off_len;
        }
        last = id;
        out_ids[o] = id;
        out_freqs[o] = r.freq;
        if (out_masks) out_masks[o] = (uint32_t)r.mask_lo;
    }
}

// numeric index blocks -> (docId, value) arrays, one thread per block (records are a dependent chain like the term codecs)
__global__ void decode_numeric_blocks_kernel(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ byte_off,
                                             const uint64_t *__restrict__ first_id, const uint32_t *__restrict__ entry_off, uint32_t nblocks,
                                             uint32_t *__restrict__ out_ids, double *__restrict__ out_values) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const uint8_t *p = bytes + byte_off[b];
    const uint32_t n = entry_off[b + 1] - entry_off[b];
    uint32_t o = entry_off[b];
    uint64_t last = first_id[b];
    for (uint32_t e = 0; e < n; e++, o++) {
        uint64_t delta;
        double v;
        p = ii_decode_numeric<false>(p, nullptr, delta, v);
        last += delta;
        out_ids[o] = (uint32_t)last;
        out_values[o] = v;
    }
}
// FilterNumericReader + the numeric iterator's one-result-per-document rule (a multi-value document has several records with
// the same docId, adjacent: the first one in range is the hit): flag, count per chunk, ordered compaction
__device__ __forceinline__ bool numeric_keep(const uint32_t *ids, const double *values, uint32_t i, double mn, double mx, bool mni, bool mxi) {
    if (!ii_numeric_in_range(values[i], mn, mx, mni, mxi)) return false;
    for (uint32_t k = i; k > 0 && ids[k - 1] == ids[i]; k--)
        if (ii_numeric_in_range(values[k - 1], mn, mx, mni, mxi)) return false; // an earlier record of the same document already hit
    return true;
}
__global__ void numeric_flags_kernel(const uint32_t *__restrict__ ids, const double *__restrict__ values, uint32_t n, double mn, double mx,
                                     int mni, int mxi, uint32_t *__restrict__ chunk_counts) {
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t c = 0;
    for (uint32_t i = threadIdx.x; i < 1024u; i += blockDim.x)
        if (base + i < n && numeric_keep(ids, values, base + i, mn, mx, mni, mxi)) c++;
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) chunk_counts[blockIdx.x] = s_cnt;
}
__global__ void numeric_compact_kernel(const uint32_t *__restrict__ ids, const double *__restrict__ values, uint32_t n, double mn, double mx,
                                       int mni, int mxi, const uint32_t *__restrict__ chunk_off, uint32_t *__restrict__ out_ids,
                                       uint32_t *__restrict__ out_freqs) {
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t o = chunk_off[blockIdx.x];
    const int lane = threadIdx.x;
    for (uint32_t i0 = 0; i0 < 1024u; i0 += 32) {
        const uint32_t i = base + i0 + lane;
        const bool keep = i < n && numeric_keep(ids, values, i, mn, mx, mni, mxi);
        const uint32_t mask = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const uint32_t dst = o + __popc(mask & ((1u << lane) - 1u));
            out_ids[dst] = ids[i];
            out_freqs[dst] = 1; // RSIndexResult::build_numeric: freq 1
        }
        o += __popc(mask);
    }
}

// keep records with (mask & filter) != 0, in order: flags -> scan done by the caller (scan_kernel)
__global__ void mask_flags_kernel(const uint32_t *__restrict__ masks, uint32_t n, uint32_t filter,
                                  uint32_t *__restrict__ chunk_counts) {
    // one CTA per 1024 entries
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t c = 0;
    for (uint32_t i = threadIdx.x; i < 1024u; i += blockDim.x)
        if (base + i < n && (masks[base + i] & filter)) c++;
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) chunk_counts[blockIdx.x] = s_cnt;
}
__global__ void mask_compact_kernel(const uint32_t *__restrict__ ids, const uint32_t *__restrict__ freqs,
                                    const uint32_t *__restrict__ masks, uint32_t n, uint32_t filter,
                                    const uint32_t *__restrict__ chunk_off, uint32_t *__restrict__ out_ids,
                                    uint32_t *__restrict__ out_freqs) {
    // one warp-serial pass per 1024-entry chunk keeps the order (chunks are small)
    if (threadIdx.x != 0) return;
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t o = chunk_off[blockIdx.x];
    for (uint32_t i = 0; i < 1024u && base + i < n; i++)
        if (masks[base + i] & filter) {
            out_ids[o] = ids[base + i];
            out_freqs[o] = freqs[base + i];
            o++;
        }
}

// ------------------------------------------------------------------------------------------------
// intersection
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t *a, uint32_t lo, uint32_t hi, uint32_t key) {
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (a[mid] < key)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// lower_bound of kIIItems keys at once over the same [0, range) of a shared-memory window: a fixed trip count and no
// data-dependent branches, so the compiler interleaves the independent chains (one LDS latency per step for all of a thread's
// entries, where a per-entry loop waits on each compare)
template <int N>
__device__ __forceinline__ void lower_bound_lockstep(const uint32_t *w, uint32_t range, const uint32_t (&key)[N], uint32_t (&out)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) out[i] = 0;
    if (range == 0) return;
    uint32_t n = range;
    while (n > 1) {
        const uint32_t half = n >> 1;
#pragma unroll
        for (int i = 0; i < N; i++) out[i] += (w[out[i] + half - 1] < key[i]) ? half : 0u;
        n -= half;
    }
#pragma unroll
    for (int i = 0; i < N; i++) out[i] += (w[out[i]] < key[i]) ? 1u : 0u;
}

// asynchronous 4-byte copies global -> shared (LDGSTS): a window copy written as `sB[t] = B[t]` in a loop waits for every load
// before the next one is issued, so the staging loops serialise on load latency; with cp.async all of a thread's copies are in
// flight at once and the CTA waits once
__device__ __forceinline__ void cp_async4(uint32_t *smem_dst, const uint32_t *gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// lower_bound by a whole warp: 32 pivots per round instead of one dependent load per bisection step
// (the probed list has up to 10^7 entries in HBM: 5 rounds of latency instead of 23)
__device__ __forceinline__ uint32_t warp_lower_bound_u32(const uint32_t *a, uint32_t lo, uint32_t hi, uint32_t key, int lane) {
    while (hi - lo > 32) {
        const uint32_t span = hi - lo;
        // pivots p_i = lo + (i+1)*span/33, i = 0..31 (strictly inside (lo, hi))
        const uint32_t p = lo + (uint32_t)(((uint64_t)(lane + 1) * span) / 33);
        const bool less = a[p] < key;
        const uint32_t m = __ballot_sync(0xffffffffu, less);
        const int nless = __popc(m); // pivots are ascending, so the set bits are a prefix
        const uint32_t new_lo = nless ? __shfl_sync(0xffffffffu, p, nless - 1) + 1 : lo;
        const uint32_t new_hi = nless < 32 ? __shfl_sync(0xffffffffu, p, nless) : hi;
        lo = new_lo;
        hi = new_hi;
    }
    const uint32_t idx = lo + lane;
    const bool less = idx < hi && a[idx] < key;
    return lo + __popc(__ballot_sync(0xffffffffu, less));
}

// One list of a CTA's AND probe: its docIds, exact length, mode (0 required, 1 NOT, 2 OPTIONAL) and the nullable row that
// receives the position of every driving entry inside it (pos[e] for entry e of the driving list)
struct ProbeList {
    const uint32_t *ids;
    uint32_t len;
    int mode;
    uint32_t *pos;
};
// The k-way AND of one CTA, shared by intersect_kernel and ifb_probe_kernel: each thread's kIIItems consecutive entries e0 + i
// of the driving list (doc / alive) against lists 1 .. n-1 (list_of(j) -> ProbeList).  For every list, warps 0 and 1 find the
// window of docIds [a_lo, a_hi] with a warp-wide lower bound, the window is staged in shared memory when it fits, and each
// entry's lower bound runs there.  Stops once no entry of the CTA is alive.
template <typename ListOf>
__device__ __forceinline__ void and_probe(const uint32_t (&doc)[kIIItems], bool (&alive)[kIIItems], uint32_t e0, uint32_t a_lo, uint32_t a_hi,
                                          uint32_t n, ListOf list_of, uint32_t *sB, uint32_t &s_lo, uint32_t &s_hi) {
    for (uint32_t j = 1; j < n; j++) {
        const ProbeList L = list_of(j);
        const uint32_t *B = L.ids;
        if (threadIdx.x < 64) { // warp 0 finds the window start, warp 1 its end
            const bool first = threadIdx.x < 32;
            const uint32_t r = warp_lower_bound_u32(B, 0, L.len, first ? a_lo : a_hi + 1u, threadIdx.x & 31); // a_hi < 2^32-1
            if ((threadIdx.x & 31) == 0) *(first ? &s_lo : &s_hi) = r;
        }
        __syncthreads();
        const uint32_t lo = s_lo, hi = s_hi, range = hi - lo;
        uint32_t *posj = L.pos;
        const int mode = L.mode;
        const bool staged = range <= (uint32_t)kIISmemElems;
        if (staged) {
            for (uint32_t t = threadIdx.x; t < range; t += kIIThreads) cp_async4(&sB[t], B + lo + t);
            cp_async_wait_all();
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < kIIItems; i++) {
            if (alive[i]) {
                uint32_t p;
                bool found;
                if (staged) {
                    p = lower_bound_u32(sB, 0, range, doc[i]);
                    found = (p < range) && sB[p] == doc[i];
                    p += lo;
                } else {
                    p = lower_bound_u32(B, lo, hi, doc[i]);
                    found = (p < hi) && B[p] == doc[i];
                }
                if (mode == 0) { // required
                    alive[i] = found;
                    if (found && posj) posj[e0 + i] = p;
                } else if (mode == 1) { // NOT: present = rejected
                    alive[i] = !found;
                } else if (posj) { // OPTIONAL: remembered where present
                    posj[e0 + i] = found ? p : 0xFFFFFFFFu;
                }
            }
        }
        bool any = false;
#pragma unroll
        for (int i = 0; i < kIIItems; i++) any |= alive[i];
        if (!__syncthreads_or(any)) break; // also fences sB before the next list reuses it
    }
}

// ordered compaction of a CTA's survivors: the rank of this thread's first survivor (it holds cnt of them) and the CTA's total
__device__ __forceinline__ uint32_t cta_survivor_rank(uint32_t cnt, uint32_t *s_warp, uint32_t &total) {
    uint32_t incl = cnt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t warp_base = 0;
    total = 0;
    for (int w = 0; w < kIIThreads / 32; w++) {
        if (w < warp) warp_base += s_warp[w];
        total += s_warp[w];
    }
    return warp_base + incl - cnt;
}

__global__ void __launch_bounds__(kIIThreads) intersect_kernel(const IntersectArgs a) {
    __shared__ uint32_t sB[kIISmemElems];
    __shared__ uint32_t s_lo, s_hi;
    __shared__ uint32_t s_warp[kIIThreads / 32];
    const uint32_t chunk = blockIdx.x;
    const uint32_t start = chunk * kIIChunk;
    const uint32_t end = min(start + (uint32_t)kIIChunk, a.len[0]);
    const uint32_t *A = a.ids[0];
    const uint32_t e0 = start + threadIdx.x * kIIItems; // blocked: a thread owns consecutive entries
    uint32_t doc[kIIItems];
    bool alive[kIIItems];
#pragma unroll
    for (int i = 0; i < kIIItems; i++) {
        alive[i] = e0 + i < end;
        doc[i] = alive[i] ? A[e0 + i] : 0xFFFFFFFFu;
    }
    and_probe(doc, alive, e0, A[start], A[end - 1], a.n,
              [&](uint32_t j) { return ProbeList{a.ids[j], a.len[j], a.mode[j], a.tmp_pos + (size_t)j * a.stride}; }, sB, s_lo, s_hi);
    uint32_t cnt = 0, total;
#pragma unroll
    for (int i = 0; i < kIIItems; i++) cnt += alive[i];
    uint32_t rank = cta_survivor_rank(cnt, s_warp, total);
#pragma unroll
    for (int i = 0; i < kIIItems; i++)
        if (alive[i]) a.tmp_idx[start + rank++] = e0 + i;
    if (threadIdx.x == 0) a.counts[chunk] = total;
}

// exclusive scan of `n` counts by one CTA; total written to *total
__global__ void __launch_bounds__(1024) scan_kernel(const uint32_t *__restrict__ counts, uint32_t n,
                                                    uint32_t *__restrict__ offsets, uint32_t *__restrict__ total) {
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = (i < n) ? counts[i] : 0;
        uint32_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        uint32_t wb = 0;
        for (int w = 0; w < warp; w++) wb += s_warp[w];
        const uint32_t carry = s_carry;
        if (i < n) offsets[i] = carry + wb + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = carry + wb + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_carry;
}

// ------------------------------------------------------------------------------------------------
// scorers — src/ext/default.c, same operations in the same order and precision
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double bm25std_leaf(double idf, double f, int doc_len, double avg, double weight) {
    const float b = 0.75f, k1 = 1.2f; // default.c:255-256
    const float one_minus_b = __fsub_rn(1.0f, b);
    const float b_len = __fmul_rn(b, (float)doc_len);
    const float k1p1 = __fadd_rn(k1, 1.0f);
    const double ratio = __ddiv_rn((double)b_len, avg);
    const double inner = __dadd_rn((double)one_minus_b, ratio);
    const double denom = __dadd_rn(f, __dmul_rn((double)k1, inner));
    const double num = __dmul_rn(__dmul_rn(__dmul_rn(weight, idf), f), (double)k1p1);
    return __ddiv_rn(num, denom); // :244
}
__device__ __forceinline__ double bm25_leaf(double idf, double f, double avg, double weight) {
    const float b = 0.5f, k1 = 1.2f; // default.c:166-167
    const float one_minus_b = __fsub_rn(1.0f, b);
    const double inner = __dadd_rn((double)one_minus_b, __dmul_rn((double)b, avg));
    const double denom = __dadd_rn(f, __dmul_rn((double)k1, inner));
    return __ddiv_rn(__dmul_rn(__dmul_rn(weight, idf), f), denom); // :173
}

// children of the aggregate in the reference's order: intersections keep the constructor's (sorted) order; a union's follows the
// active array of UnionFlat (UnionOrder: a function of the docId for a union read front to back)
struct ChildOrder {
    const uint8_t *perm; // NULL: 0..n-1
    uint32_t n;
};
__device__ __forceinline__ ChildOrder child_order_of(const UnionOrder *order, uint32_t n_children, uint32_t doc) {
    ChildOrder co{nullptr, n_children};
    if (order) {
        uint32_t e = 0;
        while (e + 1 < order->n_epochs && doc > order->bound[e]) e++;
        co.perm = order->perm[e];
        co.n = order->n_active[e];
    }
    return co;
}
// IndexResult_MinOffsetDelta without any offsets: `dist ? sqrt(dist) : num - 1`, 1 for num <= 1 (index_result.c:57-60,107)
__device__ __forceinline__ uint32_t slop_without_offsets(uint32_t num) { return num <= 1 ? 1u : num - 1u; }

__device__ double score_hit(const ScoreArgs &s, uint32_t doc, const uint32_t *freqs, size_t fstride, size_t o) {
    const float doc_score = s.doc_score ? s.doc_score[doc] : 1.0f;
    const uint32_t doc_len = s.doc_len ? s.doc_len[doc] : 0u;
    const ChildOrder co = child_order_of(s.is_union ? s.order : nullptr, s.n_children, doc);
#define II_FOR_CHILDREN(c) for (uint32_t ci_ = 0, c = 0; ci_ < co.n && ((c = co.perm ? co.perm[ci_] : ci_), true); ci_++)
#define II_W(c) (s.ext ? s.ext[c] : s.weight[c])
#define II_IDF(c) (s.ext ? s.ext[s.n_children + (c)] : s.idf[c])
#define II_BIDF(c) (s.ext ? s.ext[2 * s.n_children + (c)] : s.bm25_idf[c])
    // a nested aggregate child: its recursive value, computed over the child's own hits, through the hit's position inside it
#define II_NESTED(c) (!s.ext && s.sub[c] != nullptr)
#define II_SUB(c, dst, present)                                          \
    do {                                                                 \
        const uint32_t p_ = s.pos[(size_t)(c) * s.pstride + o];         \
        (present) = p_ != 0xFFFFFFFFu;                                   \
        if (present) (dst) = s.sub[c][p_];                               \
    } while (0)
    uint32_t slop = 1;
    if (s.scorer >= 1 && s.scorer <= 3 && !s.sub_only) { // the legacy scorers divide by GetSlop (:130-131, :226-227)
        if (s.slop) {
            slop = s.slop[o];
        } else if (s.is_union) {
            uint32_t present = 0;
            for (uint32_t c = 0; c < s.n_children; c++) present += freqs[c * fstride + o] != 0;
            slop = slop_without_offsets(present);
        } else {
            slop = slop_without_offsets(s.n_children);
        }
    }
    switch (s.scorer) {
    case 0:   // BM25STD            :253-316
    case 5: { // BM25STD.TANH       :339-359
        double ret = 0;
        II_FOR_CHILDREN(c) {
            if (II_NESTED(c)) {
                double v = 0;
                bool present;
                II_SUB(c, v, present);
                if (present) ret = __dadd_rn(ret, v);
                continue;
            }
            const uint32_t f = freqs[c * fstride + o];
            if (f) ret = __dadd_rn(ret, bm25std_leaf(II_BIDF(c), (double)f, (int)doc_len, s.avg_doc_len, II_W(c)));
        }
        ret = __dmul_rn(ret, s.agg_weight);
        if (s.sub_only) return ret;
        const double score = __dmul_rn((double)doc_score, ret);
        if (s.scorer == 5) return tanh(__dmul_rn(__ddiv_rn(1.0, (double)s.tanh_factor), score));
        return score;
    }
    case 1: { // BM25 (legacy)      :164-233
        double ret = 0;
        II_FOR_CHILDREN(c) {
            if (II_NESTED(c)) {
                double v = 0;
                bool present;
                II_SUB(c, v, present);
                if (present) ret = __dadd_rn(ret, v);
                continue;
            }
            const uint32_t f = freqs[c * fstride + o];
            if (f) ret = __dadd_rn(ret, bm25_leaf(II_IDF(c), (double)f, s.avg_doc_len, II_W(c)));
        }
        ret = __dmul_rn(ret, s.agg_weight);
        if (s.sub_only) return ret;
        const double score = __dmul_rn((double)doc_score, ret);
        if (score < s.min_score) return 0.0;
        return __ddiv_rn(score, (double)(int)slop); // `score /= slop` with an int slop
    }
    case 2:   // TFIDF              :68-146
    case 3: { // TFIDF.DOCNORM
        const uint32_t norm = (s.scorer == 2) ? (s.max_freq ? s.max_freq[doc] : 1u) : doc_len;
        if (!s.sub_only) {
            if (doc_score == 0.0f) return 0.0;
            if (norm == 0) return 0.0;
        }
        double raw = 0;
        II_FOR_CHILDREN(c) {
            if (II_NESTED(c)) {
                double v = 0;
                bool present;
                II_SUB(c, v, present);
                if (present) raw = __dadd_rn(raw, v);
                continue;
            }
            const uint32_t f = freqs[c * fstride + o];
            if (f) raw = __dadd_rn(raw, __dmul_rn(__dmul_rn(II_W(c), (double)f), II_IDF(c)));
        }
        raw = __dmul_rn(s.agg_weight, raw);
        if (s.sub_only) return raw;
        const double tfidf = __ddiv_rn(__dmul_rn((double)doc_score, raw), (double)norm);
        if (tfidf < s.min_score) return 0.0;
        return __ddiv_rn(tfidf, (double)(int)slop);
    }
    case 4: return (double)doc_score; // DOCSCORE :366-371
    case 6: {                         // DISMAX   :378-461: intersection sums, union takes the max
        double ret = 0;
        II_FOR_CHILDREN(c) {
            double leaf;
            if (II_NESTED(c)) {
                bool present;
                leaf = 0;
                II_SUB(c, leaf, present);
                if (!present) continue;
            } else {
                const uint32_t f = freqs[c * fstride + o];
                if (!f) continue;
                leaf = __dmul_rn(II_W(c), (double)f);
            }
            if (s.is_union)
                ret = (leaf > ret) ? leaf : ret;
            else
                ret = __dadd_rn(ret, leaf);
        }
        return __dmul_rn(s.agg_weight, ret);
    }
    }
#undef II_NESTED
#undef II_SUB
#undef II_FOR_CHILDREN
#undef II_W
#undef II_IDF
#undef II_BIDF
    return 0.0;
}

// survivors of the intersection -> ordered docIds, per-child freqs
__global__ void __launch_bounds__(kIIThreads) gather_kernel(const GatherArgs g) {
    const uint32_t chunk = blockIdx.x;
    const uint32_t cnt = g.counts[chunk], off = g.offsets[chunk];
    const uint32_t start = chunk * kIIChunk;
    for (uint32_t r = threadIdx.x; r < cnt; r += kIIThreads) {
        const uint32_t idx = g.tmp_idx[start + r];
        const size_t o = (size_t)off + r;
        g.out_doc[o] = g.ids0[idx];
        g.out_freq[(size_t)g.row[0] * g.fstride + o] = g.freqs[0][idx];
        if (g.out_pos) g.out_pos[(size_t)g.row[0] * g.fstride + o] = idx;
        for (uint32_t j = 1; j < g.n; j++) {
            uint32_t f = 0; // NOT children and absent OPTIONAL children are virtual results: freq 0
            uint32_t p = 0xFFFFFFFFu;
            if (g.mode[j] != 1) {
                p = g.tmp_pos[(size_t)j * g.stride + idx];
                if (g.mode[j] == 0 || p != 0xFFFFFFFFu) f = g.freqs[j][p];
            }
            if (g.out_pos) g.out_pos[(size_t)g.row[j] * g.fstride + o] = p;
            g.out_freq[(size_t)g.row[j] * g.fstride + o] = f;
        }
    }
}

__global__ void score_kernel(const ScoreArgs s, const uint32_t *__restrict__ docs, const uint32_t *__restrict__ freqs,
                             size_t fstride, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                             double *__restrict__ scores) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < m; o += (size_t)gridDim.x * blockDim.x)
        scores[o] = score_hit(s, docs[o], freqs, fstride, o);
}

// HAMMING (default.c:475-497): the byte loop of the reference is a popcount per byte; the sum is the same taken 4 bytes at a time
__global__ void hamming_kernel(const uint32_t *__restrict__ docs, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                               const uint8_t *__restrict__ payloads, const uint64_t *__restrict__ payload_off,
                               const uint8_t *__restrict__ qdata, uint32_t qlen, double *__restrict__ scores) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < m; o += (size_t)gridDim.x * blockDim.x) {
        const uint32_t doc = docs[o];
        const uint64_t b0 = payload_off[doc], b1 = payload_off[doc + 1];
        double r = 0.0;
        if (b1 > b0 && b1 - b0 == (uint64_t)qlen) { // hasPayload, len != 0, same length as the query payload
            const uint8_t *b = payloads + b0;
            uint64_t bits = 0;
            for (uint32_t i = 0; i < qlen; i++) bits += __popc((uint32_t)(qdata[i] ^ b[i]));
            r = __ddiv_rn(1.0, (double)(bits + 1));
        }
        scores[o] = r;
    }
}

// ------------------------------------------------------------------------------------------------
// union over a docId bitmap
// ------------------------------------------------------------------------------------------------
__global__ void mark_kernel(const uint32_t *__restrict__ ids, uint32_t n, uint32_t *__restrict__ bitmap) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t id = ids[i];
        atomicOr(&bitmap[id >> 5], 1u << (id & 31));
    }
}
// one warp per 32-word block
__global__ void popc_kernel(const uint32_t *__restrict__ bitmap, uint32_t nwords, uint32_t *__restrict__ blocksum) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t c = (w < nwords) ? __popc(bitmap[w]) : 0;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
    if ((threadIdx.x & 31) == 0) blocksum[w >> 5] = c;
}
__global__ void expand_kernel(const uint32_t *__restrict__ bitmap, uint32_t nwords, const uint32_t *__restrict__ blockoff,
                              uint32_t *__restrict__ wordoff, uint32_t *__restrict__ out_doc) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t bits = (w < nwords) ? bitmap[w] : 0;
    const uint32_t c = __popc(bits);
    uint32_t incl = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (w >= nwords) return;
    uint32_t o = blockoff[w >> 5] + incl - c;
    wordoff[w] = o;
    while (bits) {
        const int b = __ffs(bits) - 1;
        bits &= bits - 1;
        out_doc[o++] = (w << 5) + b;
    }
}
__global__ void fill_freq_kernel(const uint32_t *__restrict__ ids, const uint32_t *__restrict__ freqs, uint32_t n,
                                 const uint32_t *__restrict__ bitmap, const uint32_t *__restrict__ wordoff,
                                 uint32_t *__restrict__ out_freq, uint32_t *__restrict__ out_pos) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t id = ids[i], w = id >> 5;
        const uint32_t rank = wordoff[w] + __popc(bitmap[w] & ((1u << (id & 31)) - 1u));
        out_freq[rank] = freqs[i];
        if (out_pos) out_pos[rank] = i;
    }
}

// ------------------------------------------------------------------------------------------------
// a batch of unions / numeric range filters: the kernels above, ragged over every list of every query (ii_kernels.h: UBList)
// ------------------------------------------------------------------------------------------------
// the table entry (a list here, a query of II_IntersectFilterBatchDevice) that owns chunk b: the last one whose first chunk is
// <= b (entries that own no chunk, such as empty lists, are not in the table)
template <typename T>
__device__ __forceinline__ uint32_t chunk_owner(const T *__restrict__ tab, uint32_t n, uint32_t b) {
    uint32_t lo = 0, hi = n; // answer in [lo, hi)
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (tab[mid].chunk0 <= b) lo = mid;
        else hi = mid;
    }
    return lo;
}
// the window bit of docId id, or false when it lies outside (never for lists whose bounds the host tracked)
__device__ __forceinline__ bool ub_bit(const UBQuery &q, uint32_t id, uint64_t &word, uint32_t &bit) {
    if (id < q.lo_word * 32u) return false;
    const uint32_t local = id - q.lo_word * 32u;
    if ((local >> 5) >= q.nwords) return false;
    word = q.blk0 * 32 + (local >> 5);
    bit = local & 31;
    return true;
}
__global__ void __launch_bounds__(256) ub_mark_kernel(const UBList *__restrict__ lists, uint32_t nlists, const UBQuery *__restrict__ qs,
                                                      uint32_t *__restrict__ bitmap, uint32_t *__restrict__ est) {
    __shared__ uint32_t s_l, s_kept;
    if (threadIdx.x == 0) {
        s_l = chunk_owner(lists, nlists, blockIdx.x);
        s_kept = 0;
    }
    __syncthreads();
    const UBList L = lists[s_l];
    const UBQuery &q = qs[L.q];
    const uint32_t base = (blockIdx.x - L.chunk0) * kUBChunk, len = L.d_len ? min(*L.d_len, L.len) : L.len;
    if (base >= len) return; // a set's chunk past its count on the device: no read of its docIds (never a numeric leaf)
    const uint32_t end = min(base + kUBChunk, len);
    uint32_t kept = 0;
    for (uint32_t i = base + threadIdx.x; i < end; i += blockDim.x) {
        if (L.values) { // a numeric leaf: only records in range mark; the first of its document counts toward num_estimated
            if (!ii_numeric_in_range(L.values[i], q.mn, q.mx, q.mni, q.mxi)) continue;
            if (numeric_keep(L.ids, L.values, i, q.mn, q.mx, q.mni, q.mxi)) kept++;
        }
        uint64_t w;
        uint32_t bit;
        if (ub_bit(q, L.ids[i], w, bit)) atomicOr(&bitmap[w], 1u << bit);
    }
    if (!L.values) return;
    atomicAdd(&s_kept, kept);
    __syncthreads();
    if (threadIdx.x == 0 && s_kept) atomicAdd(&est[L.q], s_kept);
}
// bits per 32-word block; the windows are whole blocks, so a warp never straddles two queries
__global__ void ub_popc_kernel(const uint32_t *__restrict__ bitmap, uint64_t total_words, uint32_t *__restrict__ blocksum) {
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total_words; w += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t c = __popc(bitmap[w]);
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
        if ((threadIdx.x & 31) == 0) blocksum[w >> 5] = c;
    }
}
// one CTA per query: exclusive scan of its blocks' counts, the count into len[0] (and len[1] for numeric filters and ORs over
// sets), and the set's epoch table out of the batch table
constexpr int kUBScanThreads = 1024, kUBScanItems = 8;
// exclusive scan of in[0, n) into out by one CTA of kUBScanThreads threads; returns the total to every thread
__device__ uint32_t cta_exclusive_scan(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint32_t n, uint32_t *s_warp,
                                       uint32_t &s_carry) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t t0 = 0; t0 < n; t0 += kUBScanThreads * kUBScanItems) {
        const uint32_t i0 = t0 + threadIdx.x * kUBScanItems;
        uint32_t v[kUBScanItems], sum = 0;
#pragma unroll
        for (int k = 0; k < kUBScanItems; k++) {
            v[k] = i0 + k < n ? in[i0 + k] : 0;
            sum += v[k];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = s_warp[lane], wi = w;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
                if (lane >= d) wi += t;
            }
            s_warp[lane] = wi - w; // exclusive prefix of the warps
        }
        __syncthreads();
        uint32_t o = s_carry + s_warp[warp] + incl - sum;
#pragma unroll
        for (int k = 0; k < kUBScanItems; k++) {
            if (i0 + k < n) out[i0 + k] = o;
            o += v[k];
        }
        __syncthreads(); // every thread has read s_carry and s_warp
        if (threadIdx.x == kUBScanThreads - 1) s_carry = o;
        __syncthreads();
    }
    return s_carry;
}
__global__ void __launch_bounds__(kUBScanThreads) ub_scan_kernel(const UBQuery *__restrict__ qs, const uint32_t *__restrict__ blocksum,
                                                                 uint32_t *__restrict__ blockoff, const uint32_t *__restrict__ est) {
    __shared__ uint32_t s_warp[32], s_carry;
    const UBQuery &q = qs[blockIdx.x];
    const uint32_t total = cta_exclusive_scan(blocksum + q.blk0, blockoff + q.blk0, q.nblk, s_warp, s_carry);
    if (threadIdx.x == 0) {
        q.len[0] = total;
        if (!q.sum_est) q.len[1] = est[blockIdx.x];
    }
    if (q.sum_est && threadIdx.x < 32) { // an OR over sets: the estimates still on the device (at most 1024) summed by one warp
        unsigned long long sum = 0;
        for (uint32_t i = threadIdx.x; i < q.n_est_dev; i += 32) sum += *q.est_dev[i];
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, m);
        if (threadIdx.x == 0) q.len[1] = (uint32_t)min(sum + q.est_host, 0xFFFFFFFFull);
    }
    if (q.order) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(q.order_src);
        uint32_t *dst = reinterpret_cast<uint32_t *>(q.order);
        for (uint32_t w = threadIdx.x; w < sizeof(UnionOrder) / 4; w += blockDim.x) dst[w] = src[w];
    }
}
// ascending docIds of every window: a warp per 32-word block, the query found by binary search over the windows' first blocks
__device__ __forceinline__ uint32_t ub_query_of(const UBQuery *__restrict__ qs, uint32_t nq, uint64_t blk) {
    uint32_t lo = 0, hi = nq;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (qs[mid].blk0 <= blk) lo = mid;
        else hi = mid;
    }
    return lo;
}
__global__ void ub_expand_kernel(const UBQuery *__restrict__ qs, uint32_t nq, const uint32_t *__restrict__ bitmap, uint64_t total_words,
                                 const uint32_t *__restrict__ blockoff, uint32_t *__restrict__ wordoff) {
    const int lane = threadIdx.x & 31;
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total_words; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t blk = w >> 5;
        const UBQuery &q = qs[ub_query_of(qs, nq, blk)];
        uint32_t bits = bitmap[w]; // words past the window stay clear
        const uint32_t c = __popc(bits);
        uint32_t incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        uint32_t o = blockoff[blk] + incl - c;
        if (wordoff) wordoff[w] = o;
        const uint32_t id0 = (q.lo_word + (uint32_t)(w - q.blk0 * 32)) << 5;
        while (bits) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            q.docs[o++] = id0 + b;
        }
    }
}
// full mode: rows [0, count) of every child zeroed (positions ~0) before the fill; a tile of 256 hits of one row per CTA step
__global__ void ub_clear_kernel(const UBQuery *__restrict__ qs, uint32_t nq) {
    for (uint32_t qi = blockIdx.y; qi < nq; qi += gridDim.y) {
        const UBQuery &q = qs[qi];
        const uint32_t m = *q.len, tpr = (m + 255) / 256;
        const uint64_t tiles = (uint64_t)tpr * q.n_rows;
        for (uint64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
            const uint64_t r = t / tpr;
            const uint32_t o = (uint32_t)(t - r * tpr) * 256 + threadIdx.x;
            if (o >= m) continue;
            q.freqs[r * q.cap + o] = 0;
            if (q.pos) q.pos[r * q.cap + o] = 0xFFFFFFFFu;
        }
    }
}
// full mode: every posting's freq (and position) into its child's row at the rank of its docId (as fill_freq_kernel)
__global__ void __launch_bounds__(256) ub_fill_kernel(const UBList *__restrict__ lists, uint32_t nlists, const UBQuery *__restrict__ qs,
                                                      const uint32_t *__restrict__ bitmap, const uint32_t *__restrict__ wordoff) {
    __shared__ uint32_t s_l;
    if (threadIdx.x == 0) s_l = chunk_owner(lists, nlists, blockIdx.x);
    __syncthreads();
    const UBList L = lists[s_l];
    const UBQuery &q = qs[L.q];
    const uint32_t base = (blockIdx.x - L.chunk0) * kUBChunk, end = min(base + kUBChunk, L.len);
    for (uint32_t i = base + threadIdx.x; i < end; i += blockDim.x) {
        uint64_t w;
        uint32_t bit;
        if (!ub_bit(q, L.ids[i], w, bit)) continue;
        const uint32_t rank = wordoff[w] + __popc(bitmap[w] & ((1u << bit) - 1u));
        q.freqs[L.row * q.cap + rank] = L.freqs[i];
        if (q.pos) q.pos[L.row * q.cap + rank] = i;
    }
}

// ------------------------------------------------------------------------------------------------
// a batch of filter-mode ANDs over lists and sets (ii_kernels.h: IFBChild): the probe of intersect_kernel, ragged over the
// driver chunks of every query, with each set child's length read on the device
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ifb_len(const IFBChild &c) { return c.d_len ? min(*c.d_len, c.len) : c.len; }

__global__ void __launch_bounds__(kIIThreads) ifb_probe_kernel(const IFBChild *__restrict__ children, const IFBQuery *__restrict__ qs,
                                                               uint32_t nq, uint32_t *__restrict__ surv, uint32_t *__restrict__ counts) {
    __shared__ uint32_t sB[kIISmemElems];
    __shared__ uint32_t s_lo, s_hi;
    __shared__ uint32_t s_warp[kIIThreads / 32];
    __shared__ uint32_t s_q;
    if (threadIdx.x == 0) s_q = chunk_owner(qs, nq, blockIdx.x);
    __syncthreads();
    const IFBQuery &q = qs[s_q];
    const IFBChild *ch = children + q.child0;
    const uint32_t start = (blockIdx.x - q.chunk0) * kIIChunk, n0 = ifb_len(ch[0]);
    if (start >= n0) { // past the driver's count on the device: no entry, and no read of its docIds
        if (threadIdx.x == 0) counts[blockIdx.x] = 0;
        return;
    }
    const uint32_t end = min(start + (uint32_t)kIIChunk, n0);
    const uint32_t *A = ch[0].ids;
    const uint32_t e0 = start + threadIdx.x * kIIItems;
    uint32_t doc[kIIItems];
    bool alive[kIIItems];
#pragma unroll
    for (int i = 0; i < kIIItems; i++) {
        alive[i] = e0 + i < end;
        doc[i] = alive[i] ? A[e0 + i] : 0xFFFFFFFFu;
    }
    and_probe(doc, alive, e0, A[start], A[end - 1], q.n,
              [&](uint32_t j) { return ProbeList{ch[j].ids, ifb_len(ch[j]), (int)ch[j].mode, nullptr}; }, sB, s_lo, s_hi);
    uint32_t cnt = 0, total;
#pragma unroll
    for (int i = 0; i < kIIItems; i++) cnt += alive[i];
    uint32_t rank = cta_survivor_rank(cnt, s_warp, total);
    uint32_t *out = surv + (size_t)blockIdx.x * kIIChunk;
#pragma unroll
    for (int i = 0; i < kIIItems; i++)
        if (alive[i]) out[rank++] = doc[i];
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}
// one CTA per query: exclusive scan of its chunks' counts, the count into len[0], every child's num_estimated into len[2 + slot]
// and the smallest required one into len[1]
__global__ void __launch_bounds__(kUBScanThreads) ifb_scan_kernel(const IFBChild *__restrict__ children, const IFBQuery *__restrict__ qs,
                                                                  const uint32_t *__restrict__ counts, uint32_t *__restrict__ offsets) {
    __shared__ uint32_t s_warp[32], s_carry;
    const IFBQuery &q = qs[blockIdx.x];
    const uint32_t total = cta_exclusive_scan(counts + q.chunk0, offsets + q.chunk0, q.nchunks, s_warp, s_carry);
    if (threadIdx.x >= 32) return;
    const uint32_t lane = threadIdx.x;
    uint32_t est = 0xFFFFFFFFu;
    if (lane < q.n) { // n <= kIIMaxLists = 32
        const IFBChild &c = children[q.child0 + lane];
        const uint32_t e = c.d_est ? *c.d_est : c.est;
        q.len[2 + c.slot] = e;
        if (c.mode == 0) est = e;
    }
    est = __reduce_min_sync(0xffffffffu, est);
    if (lane == 0) {
        q.len[0] = total;
        q.len[1] = est;
    }
}
// one CTA per driver chunk: its survivors to their place in the query's docIds
__global__ void __launch_bounds__(kIIThreads) ifb_expand_kernel(const IFBQuery *__restrict__ qs, uint32_t nq, const uint32_t *__restrict__ surv,
                                                                const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offsets) {
    __shared__ uint32_t s_q;
    const uint32_t m = counts[blockIdx.x];
    if (!m) return; // the whole CTA
    if (threadIdx.x == 0) s_q = chunk_owner(qs, nq, blockIdx.x);
    __syncthreads();
    const IFBQuery &q = qs[s_q];
    const uint32_t *src = surv + (size_t)blockIdx.x * kIIChunk;
    uint32_t *dst = q.docs + offsets[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < m; i += kIIThreads) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------------------
// top-N by (score desc, docId asc) — cmpByScore, src/result_processor.c:834-850
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t rank_key(double score) { // smaller key = better rank
    uint64_t u = (uint64_t)__double_as_longlong(score + 0.0);
    u = (u >> 63) ? ~u : (u | 0x8000000000000000ull); // ascending-orderable
    return ~u;                                        // descending score
}
struct Cand {
    uint64_t key;
    uint32_t id;
};
__device__ __forceinline__ bool cand_less(uint64_t ka, uint32_t ia, uint64_t kb, uint32_t ib) {
    return ka < kb || (ka == kb && ia < ib);
}

// per-warp lists in smem: keys[k], ids[k]; returns through global lists; final merge by one CTA
__global__ void __launch_bounds__(256) topn_kernel(const uint32_t *__restrict__ docs, const double *__restrict__ scores,
                                                   const uint32_t *__restrict__ d_len, uint32_t cap_len, uint32_t k,
                                                   uint64_t *__restrict__ out_keys, uint32_t *__restrict__ out_ids) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem) + (size_t)warp * k;
    uint32_t *ids = reinterpret_cast<uint32_t *>(reinterpret_cast<uint64_t *>(smem) + (size_t)8 * k) + (size_t)warp * k;
    for (uint32_t p = lane; p < k; p += 32) {
        keys[p] = 0xFFFFFFFFFFFFFFFFull;
        ids[p] = 0xFFFFFFFFu;
    }
    __syncwarp();
    uint64_t wkey = 0xFFFFFFFFFFFFFFFFull; // worst entry of this warp's list (warp-uniform)
    uint32_t wid = 0xFFFFFFFFu, wpos = 0;
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    const uint32_t gw = blockIdx.x * 8 + warp, nw = gridDim.x * 8;
    for (uint64_t base = (uint64_t)gw * 32; base < m; base += (uint64_t)nw * 32) {
        const uint32_t i = (uint32_t)base + lane;
        const bool valid = i < m;
        const uint64_t ck = valid ? rank_key(scores[i]) : 0xFFFFFFFFFFFFFFFFull;
        const uint32_t ci = valid ? docs[i] : 0xFFFFFFFFu;
        unsigned pending = __ballot_sync(0xffffffffu, valid && cand_less(ck, ci, wkey, wid));
        while (pending) {
            const int src = __ffs(pending) - 1;
            pending &= pending - 1;
            const uint64_t k2 = shfl_u64(ck, src);
            const uint32_t i2 = __shfl_sync(0xffffffffu, ci, src);
            if (!cand_less(k2, i2, wkey, wid)) continue;
            if (lane == 0) {
                keys[wpos] = k2;
                ids[wpos] = i2;
            }
            __syncwarp();
            uint64_t bk = 0;
            uint32_t bi = 0, bp = 0;
            for (uint32_t p = lane; p < k; p += 32) {
                const uint64_t kk = keys[p];
                const uint32_t ii = ids[p];
                if (!cand_less(kk, ii, bk, bi)) {
                    bk = kk;
                    bi = ii;
                    bp = p;
                }
            }
#pragma unroll
            for (int mm = 16; mm > 0; mm >>= 1) {
                const uint64_t ok = shfl_xor_u64(bk, mm);
                const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, mm);
                const uint32_t op = __shfl_xor_sync(0xffffffffu, bp, mm);
                if (cand_less(bk, bi, ok, oi) || (ok == bk && oi == bi && op < bp)) {
                    bk = ok;
                    bi = oi;
                    bp = op;
                }
            }
            wkey = bk;
            wid = bi;
            wpos = bp;
            __syncwarp(); // every lane has finished reading the list before lane 0 inserts the next candidate
        }
    }
    __syncwarp();
    for (uint32_t p = lane; p < k; p += 32) {
        out_keys[(size_t)gw * k + p] = keys[p];
        out_ids[(size_t)gw * k + p] = ids[p];
    }
}

// ------------------------------------------------------------------------------------------------
// fused batch search (II_SearchTopNBatch): two launches for the whole batch instead of a five-kernel chain with a host
// synchronisation per query (whose launch chain costs more than the work)
// ------------------------------------------------------------------------------------------------
struct ScoreAcc { // the reference's scorers evaluated child by child, in aggregate child order (src/ext/default.c)
    double ret;
};
__device__ __forceinline__ void score_child(const FusedCommon &fc, ScoreAcc &a, double weight, double idf, double bm25_idf, uint32_t f,
                                            uint32_t doc_len) {
    if (!f) return;
    switch (fc.scorer) {
    case 0:
    case 5: a.ret = __dadd_rn(a.ret, bm25std_leaf(bm25_idf, (double)f, (int)doc_len, fc.avg_doc_len, weight)); break;
    case 1: a.ret = __dadd_rn(a.ret, bm25_leaf(idf, (double)f, fc.avg_doc_len, weight)); break;
    case 2:
    case 3: a.ret = __dadd_rn(a.ret, __dmul_rn(__dmul_rn(weight, (double)f), idf)); break;
    case 6: a.ret = __dadd_rn(a.ret, __dmul_rn(weight, (double)f)); break; // DISMAX over an intersection sums
    default: break;
    }
}
// n_children: the fused path carries no term positions, so GetSlop is `children - 1` (1 for a single child); lists that do carry
// positions take the per-query chain when a legacy scorer is asked for (II_SearchTopNBatch)
__device__ __forceinline__ double score_finish(const FusedCommon &fc, const ScoreAcc &a, uint32_t doc, uint32_t doc_len, uint32_t n_children) {
    const float doc_score = fc.doc_score ? fc.doc_score[doc] : 1.0f;
    switch (fc.scorer) {
    case 0:
    case 5: {
        const double score = __dmul_rn((double)doc_score, __dmul_rn(a.ret, fc.agg_weight));
        if (fc.scorer == 5) return tanh(__dmul_rn(__ddiv_rn(1.0, (double)fc.tanh_factor), score));
        return score;
    }
    case 1: {
        const double score = __dmul_rn((double)doc_score, __dmul_rn(a.ret, fc.agg_weight));
        return (score < 0.0) ? 0.0 : __ddiv_rn(score, (double)(int)slop_without_offsets(n_children)); // minScore = 0 on this path
    }
    case 2:
    case 3: {
        if (doc_score == 0.0f) return 0.0;
        const uint32_t norm = (fc.scorer == 2) ? (fc.max_freq ? fc.max_freq[doc] : 1u) : doc_len;
        if (norm == 0) return 0.0;
        const double tfidf = __ddiv_rn(__dmul_rn((double)doc_score, __dmul_rn(fc.agg_weight, a.ret)), (double)norm);
        return (tfidf < 0.0) ? 0.0 : __ddiv_rn(tfidf, (double)(int)slop_without_offsets(n_children));
    }
    case 4: return (double)doc_score;
    case 6: return __dmul_rn(fc.agg_weight, a.ret);
    }
    return 0.0;
}

// ascending bitonic sort of n (power of two) (key, id) pairs in shared memory by one CTA: (key asc, id asc)
__device__ __forceinline__ void bitonic_sort_pairs(uint64_t *keys, uint32_t *ids, uint32_t n) {
    for (uint32_t size = 2; size <= n; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (uint32_t t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = ((lo & size) == 0);
                const uint64_t ka = keys[lo], kb = keys[hi];
                const uint32_t ia = ids[lo], ib = ids[hi];
                const bool a_gt_b = cand_less(kb, ib, ka, ia);
                if (a_gt_b == up) {
                    keys[lo] = kb, keys[hi] = ka;
                    ids[lo] = ib, ids[hi] = ia;
                }
            }
        }
    }
    __syncthreads();
}

// Pre-pass of the fused search: which query owns a work item, and for every (item, other child j) the window [lo, hi) of child
// j that can hold the item's docIds.  Locating the windows inside fused_and_kernel with two warp-wide searches per list
// behind a barrier each puts several dependent HBM round trips per list on the critical path of every CTA.  Here every search
// is one thread and all of them are in flight at once.
__global__ void fused_itemq_kernel(const FusedQuery *__restrict__ queries, uint32_t nq, uint32_t *__restrict__ item_q) {
    const uint32_t q = blockIdx.x;
    if (q >= nq) return;
    const uint32_t i0 = queries[q].item0, nc = queries[q].nchunks;
    for (uint32_t t = threadIdx.x; t < nc; t += blockDim.x) item_q[i0 + t] = q;
}
__global__ void __launch_bounds__(256) fused_window_kernel(const FusedQuery *__restrict__ queries, const uint32_t *__restrict__ item_q,
                                                           uint32_t total_items, uint32_t max_others, uint2 *__restrict__ win) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (uint64_t)total_items * max_others) return;
    const uint32_t item = (uint32_t)(g / max_others), j = (uint32_t)(g % max_others) + 1;
    const FusedQuery &Q = queries[item_q[item]];
    if (j >= Q.n) return;
    const uint32_t start = (item - Q.item0) * kIIChunk;
    const uint32_t end = min(start + (uint32_t)kIIChunk, Q.len[0]);
    const uint32_t *A = Q.ids[0], *B = Q.ids[j];
    const uint32_t k_lo = A[start], k_hi = A[end - 1] + 1u; // docIds are < 2^32 - 1
    // the two lower bounds advance in lockstep: two independent loads per round
    uint32_t lo0 = 0, hi0 = Q.len[j], lo1 = 0, hi1 = Q.len[j];
    while (lo0 < hi0 || lo1 < hi1) {
        const uint32_t m0 = lo0 + ((hi0 - lo0) >> 1), m1 = lo1 + ((hi1 - lo1) >> 1);
        const uint32_t v0 = lo0 < hi0 ? B[m0] : 0u, v1 = lo1 < hi1 ? B[m1] : 0u;
        if (lo0 < hi0) {
            if (v0 < k_lo)
                lo0 = m0 + 1;
            else
                hi0 = m0;
        }
        if (lo1 < hi1) {
            if (v1 < k_hi)
                lo1 = m1 + 1;
            else
                hi1 = m1;
        }
    }
    win[(size_t)item * (kFusedMaxLists - 1) + (j - 1)] = make_uint2(lo0, lo1);
}

// kN = the largest child count of the batch, rounded up to {2, 3, 4, 8}: the loops over the children unroll to kN, so the
// common 3-term batch carries a third of the code and of the per-entry position registers of the 8-child build
template <int kN>
__global__ void __launch_bounds__(kIIThreads, (kN <= 3 ? 5 : 4)) fused_and_kernel(const FusedQuery *__restrict__ queries, const uint32_t *__restrict__ item_q,
                                                               const uint2 *__restrict__ win, const FusedCommon fc, uint32_t top_n,
                                                               uint64_t *__restrict__ cand_keys, uint32_t *__restrict__ cand_ids,
                                                               uint32_t *__restrict__ hits, uint32_t *__restrict__ cand_fill) {
    __shared__ uint32_t sB[kIISmemElems];
    __shared__ uint32_t s_base;
    __shared__ uint64_t s_keys[kIIChunk];
    __shared__ uint32_t s_ids[kIIChunk];
    __shared__ uint32_t s_warp[kIIThreads / 32];
    const uint32_t item = blockIdx.x;
    const uint32_t q = item_q[item];
    const FusedQuery &Q = queries[q];
    const uint32_t n = Q.n;
    const uint32_t chunk = item - Q.item0;
    const uint32_t start = chunk * kIIChunk;
    const uint32_t end = min(start + (uint32_t)kIIChunk, Q.len[0]);
    const uint32_t *A = Q.ids[0];
    uint32_t doc[kIIItems], pos[kN - 1][kIIItems];
    bool alive[kIIItems];
#pragma unroll
    for (int i = 0; i < kIIItems; i++) {
        const uint32_t idx = start + threadIdx.x * kIIItems + i; // blocked: a thread owns consecutive entries
        alive[i] = idx < end;
        doc[i] = alive[i] ? A[idx] : 0xFFFFFFFFu;
    }
    // the windows of the other children (block-uniform), and where each would sit in shared memory
    uint32_t w_lo[kN - 1], w_off[kN - 1], w_len[kN - 1];
    uint32_t total_range = 0;
    bool all_fit = true;
#pragma unroll
    for (int j = 1; j < kN; j++) {
        w_lo[j - 1] = w_off[j - 1] = w_len[j - 1] = 0;
        if (j < (int)n) {
            const uint2 w = win[(size_t)item * (kFusedMaxLists - 1) + (j - 1)];
            w_lo[j - 1] = w.x;
            w_len[j - 1] = w.y - w.x;
            w_off[j - 1] = total_range;
            all_fit = all_fit && w_len[j - 1] <= (uint32_t)kIISmemElems && total_range + w_len[j - 1] <= (uint32_t)kIISmemElems;
            if (all_fit) total_range += w_len[j - 1];
        }
    }
    if (all_fit) {
        // every window at once: one round of loads, one barrier, then each entry walks the children on its own
#pragma unroll
        for (int j = 1; j < kN; j++)
            if (j < (int)n) {
                const uint32_t *B = Q.ids[j] + w_lo[j - 1];
                for (uint32_t t = threadIdx.x; t < w_len[j - 1]; t += kIIThreads) cp_async4(&sB[w_off[j - 1] + t], B + t);
            }
        cp_async_wait_all();
        __syncthreads();
#pragma unroll
        for (int j = 1; j < kN; j++)
            if (j < (int)n) {
                const uint32_t *W = sB + w_off[j - 1];
                const uint32_t range = w_len[j - 1];
                uint32_t p[kIIItems];
                lower_bound_lockstep<kIIItems>(W, range, doc, p);
#pragma unroll
                for (int i = 0; i < kIIItems; i++) {
                    alive[i] = alive[i] && (p[i] < range) && W[min(p[i], range ? range - 1 : 0u)] == doc[i];
                    pos[j - 1][i] = w_lo[j - 1] + p[i];
                }
            }
    } else {
        // a window larger than the staging buffer (a short list against a much longer one): list by list, large windows
        // searched in place
        bool any_alive = true;
#pragma unroll
        for (int j = 1; j < kN; j++) {
            if (j >= (int)n || !any_alive) break;
            const uint32_t *B = Q.ids[j];
            const uint32_t lo = w_lo[j - 1], range = w_len[j - 1], hi = lo + range;
            if (range <= (uint32_t)kIISmemElems) {
                for (uint32_t t = threadIdx.x; t < range; t += kIIThreads) cp_async4(&sB[t], B + lo + t);
                cp_async_wait_all();
                __syncthreads();
                uint32_t p[kIIItems];
                lower_bound_lockstep<kIIItems>(sB, range, doc, p);
#pragma unroll
                for (int i = 0; i < kIIItems; i++) {
                    alive[i] = alive[i] && (p[i] < range) && sB[min(p[i], range ? range - 1 : 0u)] == doc[i];
                    pos[j - 1][i] = lo + p[i];
                }
            } else {
                // a window far longer than the chunk (a rare term against a frequent one): kPivots evenly spaced entries of the
                // window go to shared memory, every entry first finds its bucket there (no HBM latency), then finishes inside
                // the bucket with its searches advancing in lockstep (one round trip per step for all of a thread's entries
                // instead of one per entry per step)
                constexpr uint32_t kPivots = 2048;
                const uint32_t step = (range + kPivots - 1) / kPivots; // bucket b = [lo + b*step, lo + (b+1)*step)
                const uint32_t nbuckets = (range + step - 1) / step;
                for (uint32_t t = threadIdx.x; t < nbuckets; t += kIIThreads) cp_async4(&sB[t], B + lo + (size_t)t * step); // first entry of bucket t
                cp_async_wait_all();
                __syncthreads();
                uint32_t l[kIIItems], h[kIIItems];
#pragma unroll
                for (int i = 0; i < kIIItems; i++) {
                    l[i] = h[i] = 0;
                    if (alive[i]) {
                        // last bucket whose first entry is <= doc: upper_bound - 1; the bucket before the first one cannot match
                        uint32_t a = 0, b = nbuckets;
                        while (a < b) {
                            const uint32_t mid = a + ((b - a) >> 1);
                            if (sB[mid] <= doc[i])
                                a = mid + 1;
                            else
                                b = mid;
                        }
                        if (a == 0) {
                            alive[i] = false; // below the window's first entry
                        } else {
                            l[i] = lo + (a - 1) * step;
                            h[i] = min(l[i] + step, hi);
                        }
                    }
                }
                bool more = true;
                while (more) {
                    uint32_t mid[kIIItems], v[kIIItems];
#pragma unroll
                    for (int i = 0; i < kIIItems; i++) {
                        mid[i] = l[i] + ((h[i] - l[i]) >> 1);
                        v[i] = (alive[i] && l[i] < h[i]) ? B[mid[i]] : 0u;
                    }
                    more = false;
#pragma unroll
                    for (int i = 0; i < kIIItems; i++)
                        if (alive[i] && l[i] < h[i]) {
                            if (v[i] < doc[i])
                                l[i] = mid[i] + 1;
                            else
                                h[i] = mid[i];
                            more |= l[i] < h[i];
                        }
                }
                uint32_t fv[kIIItems];
#pragma unroll
                for (int i = 0; i < kIIItems; i++) fv[i] = (alive[i] && l[i] < hi) ? B[l[i]] : 0xFFFFFFFFu;
#pragma unroll
                for (int i = 0; i < kIIItems; i++)
                    if (alive[i]) {
                        alive[i] = l[i] < hi && fv[i] == doc[i];
                        pos[j - 1][i] = l[i];
                    }
            }
            bool any = false;
#pragma unroll
            for (int i = 0; i < kIIItems; i++) any |= alive[i];
            any_alive = __syncthreads_or(any); // also fences sB before the next list reuses it
        }
    }
    // score the survivors, child by child in aggregate order
    uint32_t cnt = 0;
    uint64_t key[kIIItems];
#pragma unroll
    for (int i = 0; i < kIIItems; i++) {
        key[i] = 0xFFFFFFFFFFFFFFFFull;
        if (!alive[i]) continue;
        cnt++;
        const uint32_t d = doc[i];
        const uint32_t dl = fc.doc_len ? fc.doc_len[d] : 0u;
        ScoreAcc acc{0.0};
        score_child(fc, acc, Q.weight[0], Q.idf[0], Q.bm25_idf[0], Q.freqs[0][start + threadIdx.x * kIIItems + i], dl);
#pragma unroll
        for (int j = 1; j < kN; j++)
            if (j < (int)n) score_child(fc, acc, Q.weight[j], Q.idf[j], Q.bm25_idf[j], Q.freqs[j][pos[j - 1][i]], dl);
        key[i] = rank_key(score_finish(fc, acc, d, dl, n));
    }
    // ordered compaction of (key, docId) into shared memory, then the CTA's best top_n
    uint32_t incl = cnt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, dd);
        if (lane >= dd) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t warp_base = 0, total = 0;
    for (int w = 0; w < kIIThreads / 32; w++) {
        if (w < warp) warp_base += s_warp[w];
        total += s_warp[w];
    }
    uint32_t rank = warp_base + incl - cnt;
#pragma unroll
    for (int i = 0; i < kIIItems; i++)
        if (alive[i]) {
            s_keys[rank] = key[i];
            s_ids[rank] = doc[i];
            rank++;
        }
    __syncthreads();
    if (total > top_n) { // more survivors than the query keeps: the CTA's best top_n (the per-query pass takes lists in any order)
        const uint32_t nsort = max(32u, next_pow2(total));
        for (uint32_t t = total + threadIdx.x; t < nsort; t += kIIThreads) s_keys[t] = 0xFFFFFFFFFFFFFFFFull, s_ids[t] = 0xFFFFFFFFu;
        bitonic_sort_pairs(s_keys, s_ids, nsort); // entry syncs inside
    }
    // the CTA's candidates go behind those of the query's other items: a compact list per query (at most top_n per item, so the
    // query's nchunks * top_n slots always suffice); their order is whatever the atomics make it, the per-query pass sorts
    const uint32_t keep = min(total, top_n);
    if (threadIdx.x == 0 && total) {
        s_base = atomicAdd(&cand_fill[q], keep);
        atomicAdd(&hits[q], total);
    }
    __syncthreads();
    const size_t qbase = (size_t)Q.item0 * top_n + s_base;
    for (uint32_t t = threadIdx.x; t < keep; t += kIIThreads) {
        cand_keys[qbase + t] = s_keys[t];
        cand_ids[qbase + t] = s_ids[t];
    }
}

// one CTA per query: best top_n of the query's compact candidate list (cand_fill[q] entries at item0 * top_n).  After the first
// fold the current top_n-th best is a threshold: candidates that cannot beat it are dropped on arrival, so a query with tens of
// thousands of candidates (three frequent terms) folds twice instead of once per 1,792 candidates
__global__ void __launch_bounds__(256) fused_topn_kernel(const FusedQuery *__restrict__ queries, uint32_t top_n,
                                                         const uint64_t *__restrict__ cand_keys, const uint32_t *__restrict__ cand_ids,
                                                         const uint32_t *__restrict__ cand_fill, uint64_t *__restrict__ out_keys,
                                                         uint32_t *__restrict__ out_ids) {
    constexpr uint32_t kTile = 1024, kPerThread = 4;
    __shared__ uint64_t s_keys[2 * kTile];
    __shared__ uint32_t s_ids[2 * kTile];
    __shared__ uint32_t s_fill;
    const FusedQuery &Q = queries[blockIdx.x];
    const size_t base = (size_t)Q.item0 * top_n;
    const uint32_t total = cand_fill[blockIdx.x];
    // running best in [0, top_n); accepted candidates are appended behind it, the buffer sorted, the head kept
    for (uint32_t t = threadIdx.x; t < top_n; t += blockDim.x) s_keys[t] = 0xFFFFFFFFFFFFFFFFull, s_ids[t] = 0xFFFFFFFFu;
    if (threadIdx.x == 0) s_fill = top_n;
    __syncthreads();
    uint32_t fill = top_n; // block-uniform, from the barriers' own counts (s_fill is only ever touched by atomics and the reset)
    uint64_t thr_key = 0xFFFFFFFFFFFFFFFFull;
    uint32_t thr_id = 0xFFFFFFFFu;
    for (uint32_t off = 0; off < total; off += blockDim.x * kPerThread) {
        uint64_t k[kPerThread];
        uint32_t id[kPerThread];
        bool ok[kPerThread];
#pragma unroll
        for (uint32_t j = 0; j < kPerThread; j++) { // all loads of the round in flight together
            const uint32_t i = off + j * blockDim.x + threadIdx.x;
            ok[j] = i < total;
            k[j] = ok[j] ? cand_keys[base + i] : 0xFFFFFFFFFFFFFFFFull;
            id[j] = ok[j] ? cand_ids[base + i] : 0xFFFFFFFFu;
        }
#pragma unroll
        for (uint32_t j = 0; j < kPerThread; j++) {
            const bool take = ok[j] && cand_less(k[j], id[j], thr_key, thr_id);
            const uint32_t m = __ballot_sync(0xffffffffu, take);
            uint32_t wbase = 0;
            if ((threadIdx.x & 31) == 0 && m) wbase = atomicAdd(&s_fill, (uint32_t)__popc(m));
            wbase = __shfl_sync(0xffffffffu, wbase, 0);
            if (take) {
                const uint32_t p = wbase + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
                s_keys[p] = k[j];
                s_ids[p] = id[j];
            }
            fill += (uint32_t)__syncthreads_count(take);
        }
        if (fill > kTile || off + blockDim.x * kPerThread >= total) { // no room for another full round, or the last one: fold
            const uint32_t nsort = max(32u, next_pow2(fill));
            for (uint32_t t = fill + threadIdx.x; t < nsort; t += blockDim.x) s_keys[t] = 0xFFFFFFFFFFFFFFFFull, s_ids[t] = 0xFFFFFFFFu;
            bitonic_sort_pairs(s_keys, s_ids, nsort); // entry syncs inside, one at the end
            thr_key = s_keys[top_n - 1];
            thr_id = s_ids[top_n - 1];
            if (threadIdx.x == 0) s_fill = top_n;
            fill = top_n;
            __syncthreads();
        }
    }
    for (uint32_t t = threadIdx.x; t < top_n; t += blockDim.x) {
        out_keys[(size_t)blockIdx.x * top_n + t] = s_keys[t];
        out_ids[(size_t)blockIdx.x * top_n + t] = s_ids[t];
    }
}

cudaError_t ii_launch_fused_search(const FusedQuery *d_queries, uint32_t nq, uint32_t total_items, uint32_t max_children, const FusedCommon &fc,
                                   uint32_t top_n, uint32_t *d_item_q, uint2 *d_win, uint64_t *d_cand_keys, uint32_t *d_cand_ids,
                                   uint32_t *d_hits, uint64_t *d_out_keys, uint32_t *d_out_ids, cudaStream_t s) {
    if (nq == 0 || top_n == 0 || top_n > (uint32_t)kFusedMaxTopN || max_children == 0 || max_children > (uint32_t)kFusedMaxLists)
        return cudaErrorInvalidValue;
    cudaError_t e = cudaMemsetAsync(d_hits, 0, (size_t)nq * 8, s); // [nq] survivors per query, then [nq] candidate fill levels
    if (e != cudaSuccess) return e;
    uint32_t *d_fill = d_hits + nq;
    if (total_items) {
        fused_itemq_kernel<<<nq, 128, 0, s>>>(d_queries, nq, d_item_q);
        if (max_children > 1) {
            const uint64_t searches = (uint64_t)total_items * (max_children - 1);
            fused_window_kernel<<<(uint32_t)((searches + 255) / 256), 256, 0, s>>>(d_queries, d_item_q, total_items, max_children - 1, d_win);
        }
        static bool carveout_set = false; // 5 CTAs x 45 KB of static shared memory per SM need (nearly) the whole carve-out
        if (!carveout_set) {
            cudaFuncSetAttribute(fused_and_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            cudaFuncSetAttribute(fused_and_kernel<3>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            cudaFuncSetAttribute(fused_and_kernel<4>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            cudaFuncSetAttribute(fused_and_kernel<kFusedMaxLists>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            carveout_set = true;
        }
        if (max_children <= 2)
            fused_and_kernel<2><<<total_items, kIIThreads, 0, s>>>(d_queries, d_item_q, d_win, fc, top_n, d_cand_keys, d_cand_ids, d_hits, d_fill);
        else if (max_children == 3)
            fused_and_kernel<3><<<total_items, kIIThreads, 0, s>>>(d_queries, d_item_q, d_win, fc, top_n, d_cand_keys, d_cand_ids, d_hits, d_fill);
        else if (max_children == 4)
            fused_and_kernel<4><<<total_items, kIIThreads, 0, s>>>(d_queries, d_item_q, d_win, fc, top_n, d_cand_keys, d_cand_ids, d_hits, d_fill);
        else
            fused_and_kernel<kFusedMaxLists><<<total_items, kIIThreads, 0, s>>>(d_queries, d_item_q, d_win, fc, top_n, d_cand_keys, d_cand_ids, d_hits,
                                                                                 d_fill);
    }
    fused_topn_kernel<<<nq, 256, 0, s>>>(d_queries, top_n, d_cand_keys, d_cand_ids, d_fill, d_out_keys, d_out_ids);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// phrase constraints: slop / in-order over the term positions of every hit
// (RS/index_result/src/core/proximity.rs: OffsetIter::Term :45-52, within_range_in_order :127-180,
//  within_range_unordered :184-220, is_within_range :262-299; called from intersection.rs:201-242)
// ------------------------------------------------------------------------------------------------
struct OffCur {
    const uint8_t *p, *end;
    uint32_t last;
};
__device__ __forceinline__ bool off_next(OffCur &c, uint32_t &pos) {
    if (c.p >= c.end) return false;
    const uint8_t *q = c.p;
    uint8_t b = *q++;
    uint32_t val = b & 0x7f;
    while (b & 0x80) { // RS/varint: 7-bit groups, most significant first, +1 per continuation
        if (q >= c.end) return false;
        val += 1;
        b = *q++;
        val = (val << 7) | (b & 0x7f);
    }
    c.p = q;
    c.last += val; // wrapping
    pos = c.last;
    return true;
}
// one thread per hit; children in AGGREGATE order (for in_order queries that is the query order: the reference does not sort
// the children of an in-order intersection, intersection.rs:110-121)
__global__ void phrase_filter_kernel(const PhraseArgs a, const uint32_t *__restrict__ d_len, uint32_t cap_len, uint32_t *__restrict__ flags) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < m; o += gridDim.x * blockDim.x) {
        OffCur it[kPhraseMaxLists];
        uint32_t n = 0;
        for (uint32_t j = 0; j < a.n; j++) {
            const uint32_t p = a.pos[(size_t)j * a.fstride + o];
            const uint32_t raw = (a.off_len[j] && p != 0xFFFFFFFFu) ? a.off_len[j][p] : 0u; // virtual results carry no offsets
            if (raw) { // has_offsets (a nested aggregate: by its kind mask, bit 31, whatever the stream holds)
                const uint32_t len = raw & ~kIIOffLenHas;
                it[n].p = a.bytes[j] + a.off_pos[j][p];
                it[n].end = it[n].p + len;
                it[n].last = 0;
                n++;
            }
        }
        bool ok;
        if (a.n <= 1 || n <= 1) {
            ok = true;
        } else if (a.in_order) {
            uint32_t positions[kPhraseMaxLists];
            for (uint32_t i = 0; i < n; i++) positions[i] = 0;
            ok = false;
            bool done = false;
            while (!done) {
                int32_t span = 0;
                bool over = false;
                for (uint32_t i = 0; i < n; i++) {
                    uint32_t pos;
                    if (i == 0) {
                        if (!off_next(it[0], pos)) {
                            done = true;
                            break;
                        }
                    } else {
                        pos = positions[i];
                    }
                    const uint32_t last_pos = i == 0 ? 0u : positions[i - 1];
                    bool eof = false;
                    while (pos < last_pos)
                        if (!off_next(it[i], pos)) {
                            eof = true;
                            break;
                        }
                    if (eof) {
                        done = true;
                        break;
                    }
                    positions[i] = pos;
                    if (i > 0) {
                        span += (int32_t)pos - (int32_t)last_pos - 1;
                        if (span > 0 && (uint32_t)span > a.max_slop) {
                            over = true;
                            break;
                        }
                    }
                }
                if (done) break;
                if (!over) {
                    ok = true;
                    break;
                }
            }
        } else {
            uint32_t positions[kPhraseMaxLists];
            ok = false;
            bool primed = true;
            for (uint32_t i = 0; i < n; i++) primed = primed && off_next(it[i], positions[i]);
            if (primed) {
                uint32_t max_pos = 0;
                for (uint32_t i = 0; i < n; i++)
                    if (positions[i] >= max_pos) max_pos = positions[i];
                for (;;) {
                    uint32_t min_pos = 0xFFFFFFFFu, min_idx = 0;
                    for (uint32_t i = 0; i < n; i++)
                        if (positions[i] < min_pos) {
                            min_pos = positions[i];
                            min_idx = i;
                        }
                    if (min_pos != max_pos) {
                        const int32_t span = (int32_t)max_pos - (int32_t)min_pos - ((int32_t)n - 1);
                        if (span < 0 || (uint32_t)span <= a.max_slop) {
                            ok = true;
                            break;
                        }
                    }
                    uint32_t np;
                    if (!off_next(it[min_idx], np)) break;
                    positions[min_idx] = np;
                    if (np > max_pos) max_pos = np;
                }
            }
        }
        flags[o] = ok ? 1u : 0u;
    }
}
// per 1024-entry chunk: how many flagged
__global__ void flag_count_kernel(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                                  uint32_t *__restrict__ chunk_counts) {
    __shared__ uint32_t s_cnt;
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t c = 0;
    for (uint32_t i = threadIdx.x; i < 1024u; i += blockDim.x)
        if (base + i < m && flags[base + i]) c++;
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) chunk_counts[blockIdx.x] = s_cnt;
}
// ordered compaction of docs, the n freq rows and (optionally) the n posting-position rows (one warp per chunk keeps the order
// with ballots)
__global__ void flag_compact_kernel(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                                    const uint32_t *__restrict__ chunk_off, const uint32_t *__restrict__ docs,
                                    const uint32_t *__restrict__ freqs, const uint32_t *__restrict__ pos, uint32_t n, size_t fstride,
                                    uint32_t *__restrict__ out_docs, uint32_t *__restrict__ out_freqs, uint32_t *__restrict__ out_pos,
                                    size_t out_fstride) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    const uint32_t base = blockIdx.x * 1024u;
    uint32_t o = chunk_off[blockIdx.x];
    const int lane = threadIdx.x;
    for (uint32_t i0 = 0; i0 < 1024u; i0 += 32) {
        const uint32_t i = base + i0 + lane;
        const bool keep = i < m && flags[i];
        const uint32_t mask = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const uint32_t dst = o + __popc(mask & ((1u << lane) - 1u));
            out_docs[dst] = docs[i];
            for (uint32_t j = 0; j < n; j++) {
                out_freqs[(size_t)j * out_fstride + dst] = freqs[(size_t)j * fstride + i];
                if (out_pos) out_pos[(size_t)j * out_fstride + dst] = pos[(size_t)j * fstride + i];
            }
        }
        o += __popc(mask);
    }
}

cudaError_t ii_launch_phrase_filter(const PhraseArgs &a, const uint32_t *d_len, uint32_t cap_len, uint32_t *d_flags, uint32_t *d_counts,
                                    uint32_t *d_offsets, uint32_t *d_total, const uint32_t *d_docs, const uint32_t *d_freqs, size_t fstride,
                                    uint32_t *d_out_docs, uint32_t *d_out_freqs, uint32_t *d_out_pos, size_t out_fstride, cudaStream_t s) {
    if (!cap_len) return cudaMemsetAsync(d_total, 0, 4, s);
    const uint32_t chunks = (cap_len + 1023) / 1024;
    phrase_filter_kernel<<<std::max(1u, std::min((cap_len + 127) / 128, 132u * 16)), 128, 0, s>>>(a, d_len, cap_len, d_flags);
    flag_count_kernel<<<chunks, 256, 0, s>>>(d_flags, d_len, cap_len, d_counts);
    scan_kernel<<<1, 1024, 0, s>>>(d_counts, chunks, d_offsets, d_total);
    flag_compact_kernel<<<chunks, 32, 0, s>>>(d_flags, d_len, cap_len, d_offsets, d_docs, d_freqs, a.pos, a.n, fstride, d_out_docs, d_out_freqs,
                                              d_out_pos, out_fstride);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// GetSlop: IndexResult_MinOffsetDelta (src/index_result/index_result.c:51-108) per hit
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t off_next_or_eof(OffCur &c) { // RSOffsetIterator::Next: RS_OFFSETVECTOR_EOF at the end
    uint32_t p;
    return off_next(c, p) ? p : 0xFFFFFFFFu;
}
__global__ void min_offset_delta_kernel(const SlopArgs a, const uint32_t *__restrict__ docs, const uint32_t *__restrict__ d_len,
                                        uint32_t cap_len, uint32_t *__restrict__ slop) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < m; o += gridDim.x * blockDim.x) {
        const ChildOrder co = child_order_of(a.is_union ? a.order : nullptr, a.n, docs[o]);
        // the aggregate's children: all of them for an intersection (virtual results included), the present ones for a union
        uint32_t num = 0;
        int dist = 0;
        bool have_prev = false;
        OffCur prev{};
        for (uint32_t ci = 0; ci < co.n; ci++) {
            const uint32_t c = co.perm ? co.perm[ci] : ci;
            const uint32_t p = a.pos[(size_t)c * a.fstride + o];
            if (a.is_union && p == 0xFFFFFFFFu) continue; // not part of this document's aggregate
            num++;
            const uint32_t raw = (a.off_len[c] && p != 0xFFFFFFFFu) ? a.off_len[c][p] : 0u;
            if (!raw) continue; // RSIndexResult_HasOffsets :19-42: virtual results / empty offset vectors are skipped
            const uint32_t len = raw & ~kIIOffLenHas; // nested aggregates: bit 31 = counts as having offsets (kind mask)
            OffCur cur;
            cur.p = a.bytes[c] + a.off_pos[c][p];
            cur.end = cur.p + len;
            cur.last = 0;
            if (have_prev) { // the pair (previous child with offsets, this one); this one then opens the next pair (:63-104)
                OffCur v1 = prev, v2 = cur;
                uint32_t p1 = off_next_or_eof(v1), p2 = off_next_or_eof(v2);
                int cd = (int)(p2 > p1 ? p2 - p1 : p1 - p2);
                while (cd > 1 && p1 != 0xFFFFFFFFu && p2 != 0xFFFFFFFFu) {
                    const uint32_t d = p2 > p1 ? p2 - p1 : p1 - p2;
                    cd = (int)(d < (uint32_t)cd ? d : (uint32_t)cd);
                    if (p2 > p1)
                        p1 = off_next_or_eof(v1);
                    else
                        p2 = off_next_or_eof(v2);
                }
                dist += cd * cd;
            }
            prev = cur;
            have_prev = true;
        }
        uint32_t r;
        if (num <= 1)
            r = 1;
        else
            r = dist ? (uint32_t)(int)sqrt((double)dist) : num - 1;
        slop[o] = r;
    }
}
cudaError_t ii_launch_min_offset_delta(const SlopArgs &a, const uint32_t *d_docs, const uint32_t *d_len, uint32_t cap_len,
                                       uint32_t *d_slop, cudaStream_t s) {
    if (!cap_len) return cudaSuccess;
    min_offset_delta_kernel<<<std::max(1u, std::min((cap_len + 127) / 128, 132u * 16)), 128, 0, s>>>(a, d_docs, d_len, cap_len, d_slop);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// nested aggregates: summed freqs and merged term positions of every hit
// ------------------------------------------------------------------------------------------------
__global__ void sum_freq_rows_kernel(const uint32_t *__restrict__ freqs, uint32_t n, size_t fstride, const uint32_t *__restrict__ d_len,
                                     uint32_t cap_len, uint32_t *__restrict__ out) {
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < m; o += gridDim.x * blockDim.x) {
        uint32_t t = 0;
        for (uint32_t j = 0; j < n; j++) t += freqs[(size_t)j * fstride + o];
        out[o] = t;
    }
}
cudaError_t ii_launch_sum_freq_rows(const uint32_t *d_freqs, uint32_t n, size_t fstride, const uint32_t *d_len, uint32_t cap_len,
                                    uint32_t *d_out, cudaStream_t s) {
    if (!cap_len) return cudaSuccess;
    sum_freq_rows_kernel<<<std::max(1u, std::min((cap_len + 255) / 256, 132u * 8)), 256, 0, s>>>(d_freqs, n, fstride, d_len, cap_len, d_out);
    return cudaGetLastError();
}

constexpr uint32_t kMergeChunk = 256;
// is child c part of hit o's aggregate, and as what kind of result
__device__ __forceinline__ uint32_t merge_child_tag(const MergeOffsetsArgs &a, uint32_t c, uint32_t o, uint32_t &p) {
    p = a.pos ? a.pos[(size_t)c * a.fstride + o] : 0u;
    const bool there = a.pos ? p != 0xFFFFFFFFu : a.freqs[(size_t)c * a.fstride + o] != 0;
    if (a.is_union) return there ? a.tag[c] : 0u; // a union's aggregate holds the matching children only
    return there ? a.tag[c] : 8u;                  // NOT / absent OPTIONAL children of an intersection are virtual results
}
__global__ void __launch_bounds__(kMergeChunk) merge_bounds_kernel(const MergeOffsetsArgs a, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                                                                   uint32_t *__restrict__ ub, uint32_t *__restrict__ chunk_sum,
                                                                   unsigned long long *__restrict__ total64) {
    __shared__ uint32_t s_sum;
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    if (threadIdx.x == 0) s_sum = 0;
    __syncthreads();
    const uint32_t o = blockIdx.x * kMergeChunk + threadIdx.x;
    uint32_t b = 0;
    if (o < m) {
        for (uint32_t c = 0; c < a.n; c++) {
            uint32_t p;
            const uint32_t tag = merge_child_tag(a, c, o, p);
            if (tag && tag != 8u && a.off_len[c] && a.pos) b += a.off_len[c][p] & ~kIIOffLenHas;
        }
        ub[o] = b;
    }
    if (b) atomicAdd(&s_sum, b);
    __syncthreads();
    if (threadIdx.x == 0) {
        chunk_sum[blockIdx.x] = s_sum;
        if (s_sum) atomicAdd(total64, (unsigned long long)s_sum);
    }
}
__device__ __forceinline__ uint32_t varint_put(uint32_t v, uint8_t *out) { // RS/varint: most significant group first, +1 per continuation
    uint8_t buf[5];
    int at = 4;
    buf[at] = (uint8_t)(v & 0x7f);
    while (v >>= 7) {
        v -= 1;
        buf[--at] = (uint8_t)(0x80 | (v & 0x7f));
    }
    for (int i = at; i < 5; i++) out[i - at] = buf[i];
    return (uint32_t)(5 - at);
}
__global__ void __launch_bounds__(kMergeChunk) merge_write_kernel(const MergeOffsetsArgs a, const uint32_t *__restrict__ d_len, uint32_t cap_len,
                                                                  const uint32_t *__restrict__ ub, const uint32_t *__restrict__ chunk_off,
                                                                  uint8_t *__restrict__ bytes, uint32_t *__restrict__ off_pos,
                                                                  uint32_t *__restrict__ off_len) {
    __shared__ uint32_t s_warp[kMergeChunk / 32];
    const uint32_t m = d_len ? min(*d_len, cap_len) : cap_len;
    const uint32_t o = blockIdx.x * kMergeChunk + threadIdx.x;
    const uint32_t mine = o < m ? ub[o] : 0u;
    // exclusive scan of the chunk's bounds
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t base = chunk_off[blockIdx.x];
    for (int w = 0; w < warp; w++) base += s_warp[w];
    if (o >= m) return;
    const uint32_t start = base + incl - mine;
    OffCur it[kIIMaxLists];
    uint32_t head[kIIMaxLists];
    uint32_t n = 0, mask = 0;
    for (uint32_t c = 0; c < a.n; c++) {
        uint32_t p;
        const uint32_t tag = merge_child_tag(a, c, o, p);
        mask |= tag;
        if (!tag || tag == 8u || !a.off_len[c] || !a.pos) continue;
        const uint32_t len = a.off_len[c][p] & ~kIIOffLenHas;
        if (!len) continue;
        it[n].p = a.bytes[c] + a.off_pos[c][p];
        it[n].end = it[n].p + len;
        it[n].last = 0;
        if (off_next(it[n], head[n])) n++;
    }
    uint8_t *out = bytes + start;
    uint32_t written = 0, last = 0;
    while (n) { // _aoi_Next: the first child holding the smallest look-ahead yields it and advances
        uint32_t mi = 0, mv = head[0];
        for (uint32_t i = 1; i < n; i++)
            if (head[i] < mv) {
                mv = head[i];
                mi = i;
            }
        uint8_t tmp[5];
        const uint32_t k = varint_put(mv - last, tmp);
        if (written + k > mine) break; // cannot happen for ascending streams (a merged delta never exceeds the original's)
        for (uint32_t i = 0; i < k; i++) out[written + i] = tmp[i];
        written += k;
        last = mv;
        if (!off_next(it[mi], head[mi])) { // exhausted: close the gap, keeping the children's order
            for (uint32_t i = mi + 1; i < n; i++) {
                it[i - 1] = it[i];
                head[i - 1] = head[i];
            }
            n--;
        }
    }
    off_pos[o] = start;
    // RSIndexResult_HasOffsets of an aggregate: its kind mask is neither Virtual alone nor exactly Numeric|Metric
    const bool has = mask != 8u && mask != (16u | 32u);
    off_len[o] = written | (has ? kIIOffLenHas : 0u);
}
cudaError_t ii_launch_merge_offsets_bounds(const MergeOffsetsArgs &a, const uint32_t *d_len, uint32_t cap_len, uint32_t *d_ub,
                                           uint32_t *d_chunk_sum, uint32_t *d_chunk_off, uint32_t *d_total32,
                                           unsigned long long *d_total64, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(d_total64, 0, 8, s);
    if (e != cudaSuccess || !cap_len) return e;
    const uint32_t chunks = (cap_len + kMergeChunk - 1) / kMergeChunk;
    merge_bounds_kernel<<<chunks, kMergeChunk, 0, s>>>(a, d_len, cap_len, d_ub, d_chunk_sum, d_total64);
    scan_kernel<<<1, 1024, 0, s>>>(d_chunk_sum, chunks, d_chunk_off, d_total32);
    return cudaGetLastError();
}
cudaError_t ii_launch_merge_offsets_write(const MergeOffsetsArgs &a, const uint32_t *d_len, uint32_t cap_len, const uint32_t *d_ub,
                                          const uint32_t *d_chunk_off, uint8_t *d_bytes, uint32_t *d_off_pos, uint32_t *d_off_len,
                                          cudaStream_t s) {
    if (!cap_len) return cudaSuccess;
    const uint32_t chunks = (cap_len + kMergeChunk - 1) / kMergeChunk;
    merge_write_kernel<<<chunks, kMergeChunk, 0, s>>>(a, d_len, cap_len, d_ub, d_chunk_off, d_bytes, d_off_pos, d_off_len);
    return cudaGetLastError();
}

// ================================================================================================
// launchers
// ================================================================================================
static inline uint32_t grid_for(size_t n, uint32_t threads, uint32_t cap) {
    const size_t g = (n + threads - 1) / threads;
    return (uint32_t)std::max<size_t>(1, std::min<size_t>(g, cap));
}

cudaError_t ii_launch_decode(const uint8_t *d_bytes, const uint64_t *d_byte_off, const uint64_t *d_first_id,
                             const uint32_t *d_entry_off, uint32_t nblocks, int codec, uint64_t wide_filter_lo, uint64_t wide_filter_hi,
                             uint32_t *d_ids, uint32_t *d_freqs, uint32_t *d_masks, cudaStream_t s) {
    if (!nblocks) return cudaSuccess;
    decode_blocks_kernel<<<(nblocks + 127) / 128, 128, 0, s>>>(d_bytes, d_byte_off, d_first_id, d_entry_off, nblocks, codec, wide_filter_lo,
                                                              wide_filter_hi, d_ids, d_freqs, d_masks);
    return cudaGetLastError();
}
cudaError_t ii_launch_decode_staged(const uint8_t *d_bytes, const uint32_t *d_byte_off, const uint32_t *d_first_id,
                                    const uint32_t *d_entry_off, uint32_t nblocks, int codec, uint32_t *d_ids, uint32_t *d_freqs,
                                    uint32_t *d_masks, uint32_t *d_off_pos, uint32_t *d_off_len, cudaStream_t s) {
    if (!nblocks) return cudaSuccess;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(decode_blocks_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDecodeSmem);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    decode_blocks_staged_kernel<<<(nblocks + kDecodeThreads - 1) / kDecodeThreads, kDecodeThreads, kDecodeSmem, s>>>(
        d_bytes, d_byte_off, d_first_id, d_entry_off, nblocks, codec, d_ids, d_freqs, d_masks, d_off_pos, d_off_len);
    return cudaGetLastError();
}
cudaError_t ii_launch_decode_numeric(const uint8_t *d_bytes, const uint64_t *d_byte_off, const uint64_t *d_first_id, const uint32_t *d_entry_off,
                                     uint32_t nblocks, uint32_t *d_ids, double *d_values, cudaStream_t s) {
    if (!nblocks) return cudaSuccess;
    decode_numeric_blocks_kernel<<<(nblocks + 127) / 128, 128, 0, s>>>(d_bytes, d_byte_off, d_first_id, d_entry_off, nblocks, d_ids, d_values);
    return cudaGetLastError();
}
cudaError_t ii_launch_numeric_filter(const uint32_t *d_ids, const double *d_values, uint32_t n, double mn, double mx, bool min_inclusive,
                                     bool max_inclusive, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_total, uint32_t *d_out_ids,
                                     uint32_t *d_out_freqs, cudaStream_t s) {
    if (!n) return cudaMemsetAsync(d_total, 0, 4, s);
    const uint32_t chunks = (n + 1023) / 1024;
    numeric_flags_kernel<<<chunks, 256, 0, s>>>(d_ids, d_values, n, mn, mx, min_inclusive, max_inclusive, d_counts);
    scan_kernel<<<1, 1024, 0, s>>>(d_counts, chunks, d_offsets, d_total);
    numeric_compact_kernel<<<chunks, 32, 0, s>>>(d_ids, d_values, n, mn, mx, min_inclusive, max_inclusive, d_offsets, d_out_ids, d_out_freqs);
    return cudaGetLastError();
}
cudaError_t ii_launch_mask_filter(const uint32_t *d_ids, const uint32_t *d_freqs, const uint32_t *d_masks, uint32_t n,
                                  uint32_t filter, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_total,
                                  uint32_t *d_out_ids, uint32_t *d_out_freqs, cudaStream_t s) {
    if (!n) return cudaMemsetAsync(d_total, 0, 4, s);
    const uint32_t chunks = (n + 1023) / 1024;
    mask_flags_kernel<<<chunks, 256, 0, s>>>(d_masks, n, filter, d_counts);
    scan_kernel<<<1, 1024, 0, s>>>(d_counts, chunks, d_offsets, d_total);
    mask_compact_kernel<<<chunks, 32, 0, s>>>(d_ids, d_freqs, d_masks, n, filter, d_offsets, d_out_ids, d_out_freqs);
    return cudaGetLastError();
}

cudaError_t ii_launch_intersect(const IntersectArgs &a, uint32_t nchunks, uint32_t *d_offsets, uint32_t *d_total,
                                cudaStream_t s) {
    intersect_kernel<<<nchunks, kIIThreads, 0, s>>>(a);
    scan_kernel<<<1, 1024, 0, s>>>(a.counts, nchunks, d_offsets, d_total);
    return cudaGetLastError();
}
cudaError_t ii_launch_gather(const GatherArgs &g, uint32_t nchunks, cudaStream_t s) {
    gather_kernel<<<nchunks, kIIThreads, 0, s>>>(g);
    return cudaGetLastError();
}
cudaError_t ii_launch_score(const ScoreArgs &sa, const uint32_t *d_docs, const uint32_t *d_freqs, size_t fstride,
                            const uint32_t *d_len, uint32_t cap_len, double *d_scores, cudaStream_t s) {
    if (!cap_len) return cudaSuccess;
    score_kernel<<<grid_for(cap_len, 256, 132 * 8), 256, 0, s>>>(sa, d_docs, d_freqs, fstride, d_len, cap_len, d_scores);
    return cudaGetLastError();
}
cudaError_t ii_launch_union(const uint32_t *const *d_ids, const uint32_t *const *d_freqs, const uint32_t *lens, uint32_t n,
                            uint32_t nwords, uint32_t *d_bitmap, uint32_t *d_blocksum, uint32_t *d_blockoff,
                            uint32_t *d_wordoff, uint32_t *d_total, uint32_t *d_out_doc, uint32_t *d_out_freq,
                            size_t fstride, bool want_freqs, uint32_t *d_out_pos, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(d_bitmap, 0, (size_t)nwords * 4, s);
    if (e != cudaSuccess) return e;
    for (uint32_t j = 0; j < n; j++)
        if (lens[j]) mark_kernel<<<grid_for(lens[j], 256, 132 * 8), 256, 0, s>>>(d_ids[j], lens[j], d_bitmap);
    const uint32_t nblk = (nwords + 31) / 32;
    popc_kernel<<<nblk, 32, 0, s>>>(d_bitmap, nwords, d_blocksum);
    scan_kernel<<<1, 1024, 0, s>>>(d_blocksum, nblk, d_blockoff, d_total);
    expand_kernel<<<nblk, 32, 0, s>>>(d_bitmap, nwords, d_blockoff, d_wordoff, d_out_doc);
    if (want_freqs)
        for (uint32_t j = 0; j < n; j++)
            if (lens[j])
                fill_freq_kernel<<<grid_for(lens[j], 256, 132 * 8), 256, 0, s>>>(d_ids[j], d_freqs[j], lens[j], d_bitmap, d_wordoff,
                                                                                d_out_freq + (size_t)j * fstride,
                                                                                d_out_pos ? d_out_pos + (size_t)j * fstride : nullptr);
    return cudaGetLastError();
}
cudaError_t ii_launch_union_batch(const UBList *d_lists, uint32_t nlists, uint32_t total_chunks, const UBQuery *d_q, uint32_t nq,
                                  uint64_t total_blocks, uint64_t clear_elems, uint32_t *d_est, uint32_t *d_bitmap, uint32_t *d_blocksum,
                                  uint32_t *d_blockoff, uint32_t *d_wordoff, uint32_t *launches, cudaStream_t s) {
    *launches = 0;
    if (!nq || !nlists || !total_chunks) return cudaSuccess;
    const uint64_t total_words = total_blocks * 32;
    cudaError_t e = cudaMemsetAsync(d_est, 0, (size_t)(d_bitmap - d_est + total_words) * 4, s);
    if (e != cudaSuccess) return e;
    const uint32_t wgrid = grid_for(total_words, 256, 132 * 16);
    ub_mark_kernel<<<total_chunks, 256, 0, s>>>(d_lists, nlists, d_q, d_bitmap, d_est);
    ub_popc_kernel<<<wgrid, 256, 0, s>>>(d_bitmap, total_words, d_blocksum);
    ub_scan_kernel<<<nq, kUBScanThreads, 0, s>>>(d_q, d_blocksum, d_blockoff, d_est);
    ub_expand_kernel<<<wgrid, 256, 0, s>>>(d_q, nq, d_bitmap, total_words, d_blockoff, d_wordoff);
    *launches = 4;
    if (d_wordoff) {
        const uint32_t gy = std::min<uint32_t>(nq, 65535);
        const uint32_t gx = grid_for(clear_elems, 256, std::max<uint32_t>(1, 16384 / gy));
        ub_clear_kernel<<<dim3(gx, gy), 256, 0, s>>>(d_q, nq);
        ub_fill_kernel<<<total_chunks, 256, 0, s>>>(d_lists, nlists, d_q, d_bitmap, d_wordoff);
        *launches = 6;
    }
    return cudaGetLastError();
}
cudaError_t ii_launch_filter_and_batch(const IFBChild *d_children, const IFBQuery *d_q, uint32_t nq, uint32_t total_chunks,
                                       uint32_t *d_surv, uint32_t *d_counts, uint32_t *d_offsets, cudaStream_t s) {
    if (!nq || !total_chunks) return cudaSuccess;
    ifb_probe_kernel<<<total_chunks, kIIThreads, 0, s>>>(d_children, d_q, nq, d_surv, d_counts);
    ifb_scan_kernel<<<nq, kUBScanThreads, 0, s>>>(d_children, d_q, d_counts, d_offsets);
    ifb_expand_kernel<<<total_chunks, kIIThreads, 0, s>>>(d_q, nq, d_surv, d_counts, d_offsets);
    return cudaGetLastError();
}
cudaError_t ii_launch_hamming(const uint32_t *d_docs, const uint32_t *d_len, uint32_t cap_len, const uint8_t *d_payloads,
                              const uint64_t *d_payload_off, const uint8_t *d_qdata, uint32_t qlen, double *d_scores, cudaStream_t s) {
    if (!cap_len) return cudaSuccess;
    hamming_kernel<<<grid_for(cap_len, 256, 132 * 8), 256, 0, s>>>(d_docs, d_len, cap_len, d_payloads, d_payload_off, d_qdata, qlen, d_scores);
    return cudaGetLastError();
}
// docIds 1..n with freq 1: the wildcard iterator's documents (rqe_iterators/src/wildcard.rs) as a device list
__global__ void iota_kernel(uint32_t *__restrict__ ids, uint32_t *__restrict__ freqs, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        ids[i] = i + 1;
        freqs[i] = 1;
    }
}
cudaError_t ii_launch_iota(uint32_t *d_ids, uint32_t *d_freqs, uint32_t n, cudaStream_t s) {
    if (!n) return cudaSuccess;
    iota_kernel<<<grid_for(n, 256, 132 * 8), 256, 0, s>>>(d_ids, d_freqs, n);
    return cudaGetLastError();
}
uint32_t ii_topn_lists(uint32_t m) { return grid_for(m, 256, 132 * 2) * 8; }
cudaError_t ii_launch_topn(const uint32_t *d_docs, const double *d_scores, const uint32_t *d_len, uint32_t cap_len, uint32_t k,
                           uint64_t *d_keys, uint32_t *d_ids, cudaStream_t s) {
    const uint32_t grid = grid_for(cap_len, 256, 132 * 2);
    const size_t smem = (size_t)8 * k * 12;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(topn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    topn_kernel<<<grid, 256, smem, s>>>(d_docs, d_scores, d_len, cap_len, k, d_keys, d_ids);
    return cudaGetLastError();
}

} // namespace rsb200
