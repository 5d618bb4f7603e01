// Host side of libii_b200.so: posting-list objects, block decoding, the iterator algebra entry
// points, scoring, ranking and the QueryIterator facade.  Contract: include/ii_b200.h.
#include "../../include/ii_b200.h"
#include "batch_scratch.h"
#include "ii_explain.h"
#include "ii_kernels.h"
#include "ii_codec.h"
#include <functional>

#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

using namespace rsb200;

namespace {

struct Ctx { // one per calling thread: own stream, events and pinned staging (RediSearch runs one iterator
             // tree per worker thread, so concurrent FT.SEARCHes overlap on the device)
    std::mutex mu;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr;
    uint32_t *d_total = nullptr, *h_total = nullptr;
    uint8_t *h_stage = nullptr; // grow-only pinned staging for decoded postings / top-N lists
    size_t h_stage_cap = 0;
    II_Stats stats{};
    uint8_t *stage(size_t bytes) {
        if (bytes > h_stage_cap) {
            cudaStreamSynchronize(stream);
            cudaFreeHost(h_stage);
            h_stage = nullptr;
            h_stage_cap = 0;
            const size_t cap = std::max<size_t>(bytes + bytes / 4, 1 << 20);
            if (cudaMallocHost(&h_stage, cap) != cudaSuccess) {
                cudaGetLastError();
                return nullptr;
            }
            h_stage_cap = cap;
        }
        return h_stage;
    }
    // pinned staging of the tables the device filter batches upload (filter_batch_device, II_IntersectFilterBatchDevice): a slot is
    // taken again only once its last upload has executed (cudaEventQuery; a never-recorded event counts as complete), else a new
    // slot is made — never a wait
    struct UploadSlot {
        uint8_t *h = nullptr;
        size_t cap = 0;
        cudaEvent_t ev = nullptr;
    };
    std::vector<UploadSlot> up_ring;
    UploadSlot *upload_slot(size_t bytes) {
        for (UploadSlot &u : up_ring)
            if (u.cap >= bytes && cudaEventQuery(u.ev) == cudaSuccess) return &u;
        cudaGetLastError(); // cudaErrorNotReady of a slot in flight is no failure
        UploadSlot u;
        u.cap = std::max<size_t>(2 * bytes, 64 << 10);
        if (cudaMallocHost(&u.h, u.cap) != cudaSuccess) return nullptr;
        if (cudaEventCreateWithFlags(&u.ev, cudaEventDisableTiming) != cudaSuccess) {
            cudaFreeHost(u.h);
            return nullptr;
        }
        up_ring.push_back(u);
        return &up_ring.back();
    }
    bool ok = false;
    ~Ctx() { // worker thread exits; errors after runtime teardown are harmless
        if (!ok) return;
        cudaStreamSynchronize(stream);
        for (UploadSlot &u : up_ring) {
            cudaEventDestroy(u.ev);
            cudaFreeHost(u.h);
        }
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        cudaEventDestroy(e2);
        cudaFree(d_total);
        cudaFreeHost(h_total);
        cudaFreeHost(h_stage);
        cudaStreamDestroy(stream);
        cudaGetLastError();
    }
    bool init() {
        if (ok) return true;
        int nd = 0;
        if (cudaGetDeviceCount(&nd) != cudaSuccess || nd <= 0) {
            cudaGetLastError();
            fprintf(stderr, "ii_b200: no CUDA device available; this library has no CPU fallback\n");
            return false;
        }
        if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) return false;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventCreate(&e2);
        if (cudaMalloc(&d_total, 16) != cudaSuccess || cudaMallocHost(&h_total, 16) != cudaSuccess) return false;
        int dev = 0;
        cudaGetDevice(&dev);
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t keep = UINT64_MAX; // never trim: scratch of one query is reused by the next
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        ok = true;
        return true;
    }
};
// II_SearchTopNBatch runs its queries on a pool of contexts of its own; while one of those is current, every
// helper below (dalloc / dfree / copy_sync, result-set destructors) uses its stream
static thread_local Ctx *tl_ctx_override = nullptr;
Ctx &ctx() {
    if (tl_ctx_override) return *tl_ctx_override;
    static thread_local Ctx c;
    return c;
}
struct CtxScope {
    Ctx *prev;
    explicit CtxScope(Ctx *c) : prev(tl_ctx_override) { tl_ctx_override = c; }
    ~CtxScope() { tl_ctx_override = prev; }
};

// Stream-ordered allocations from the device's default memory pool (kept warm: no cudaMalloc /
// cudaFree on the query path).  Everything is allocated, used and freed in ctx().stream order.
template <typename T>
T *dalloc(size_t n) {
    T *p = nullptr;
    if (n == 0) n = 1;
    if (cudaMallocAsync(&p, n * sizeof(T), ctx().stream) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
inline void dfree(void *p) {
    if (p) cudaFreeAsync(p, ctx().stream);
}

inline cudaError_t copy_sync(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind) {
    cudaError_t e = cudaMemcpyAsync(dst, src, bytes, kind, ctx().stream);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(ctx().stream);
}

double now_us() {
    return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

} // namespace

// device memory shared by the posting lists of one batch decode (freed when the last of them goes)
struct SharedDeviceBlock {
    void *p = nullptr;
    ~SharedDeviceBlock() { dfree(p); }
};
// an event shared by the sets that must outlive it (destroyed when the last of them goes; a pending event is released once it
// completes)
struct SharedEvent {
    cudaEvent_t ev = nullptr;
    ~SharedEvent() {
        if (ev) cudaEventDestroy(ev);
    }
};
// guards II_ResultSet::readers: one set may be an input of device filter batch calls on several threads at once
static std::mutex &readers_mu() {
    static std::mutex m;
    return m;
}

struct II_PostingList {
    uint32_t *d_ids = nullptr, *d_freqs = nullptr;
    size_t n = 0;
    size_t estimated = 0; // unfiltered unique docs (num_estimated of the leaf iterator)
    uint32_t last_id = 0;
    uint32_t first_id = 0; // a lower bound on the first docId (0 where the host does not know it): bounds the window of a union batch
    std::shared_ptr<SharedDeviceBlock> owner; // set: d_ids / d_freqs are slices of owner->p
    // term positions (Full codec, kept on request): the encoded block bytes stay on the device and every posting points at
    // its offsets payload inside them
    const uint8_t *d_bytes = nullptr;
    const uint32_t *d_off_pos = nullptr, *d_off_len = nullptr;
    std::shared_ptr<SharedDeviceBlock> bytes_owner;
    // a child that is not a term leaf: an evaluated AND / OR taking part in another aggregate (II_ResultSet_IntoChild; the
    // arrays above then belong to it), a numeric / wildcard list (result_tag)
    std::shared_ptr<struct NestedSet> nested;
    uint8_t result_tag = 4;   // RSResultData tag of the results this child yields: 4 term, 8 virtual, 16 numeric, 1 union, 2 intersection
    double sort_weight = 1.0; // intersection_sort_weight (rqe_iterators: 1 / children for an intersection, else 1)
    ~II_PostingList() {
        if (!owner && !nested) {
            dfree(d_ids);
            dfree(d_freqs);
        }
    }
};

struct II_DocTable {
    uint32_t *d_len = nullptr, *d_maxf = nullptr;
    float *d_score = nullptr;
    size_t max_doc = 0;
    uint8_t *d_payloads = nullptr;    // dmd->payload bytes of every document back to back (HAMMING scorer)
    uint64_t *d_payload_off = nullptr; // [max_doc + 2]
    ~II_DocTable() {
        dfree(d_len);
        dfree(d_maxf);
        dfree(d_score);
        dfree(d_payloads);
        dfree(d_payload_off);
    }
};

struct II_ResultSet {
    uint32_t *d_docs = nullptr, *d_freqs = nullptr; // freqs [n_children][cap]
    double *d_scores = nullptr;
    uint32_t *d_len = nullptr; // hit count on the device (valid in stream order right after the AND/OR kernels)
    size_t cap = 0, len = 0;
    uint32_t n_children = 0;
    std::vector<uint32_t> child_order; // aggregate child i = lists[child_order[i]]
    bool is_union = false, has_freqs = true, scored = false;
    // term positions of the hits, kept when a child list carries them: GetSlop of the legacy scorers walks them
    // (IndexResult_MinOffsetDelta, src/index_result/index_result.c:51-108) the first time such a scorer is asked for
    uint32_t *d_hit_pos = nullptr; // [n_children][cap] posting position of the hit inside child j (aggregate order); ~0 = virtual / absent
    uint32_t *d_slop = nullptr;    // [cap]
    struct ChildOffsets {
        const uint8_t *bytes = nullptr;
        const uint32_t *off_pos = nullptr, *off_len = nullptr;
        std::shared_ptr<SharedDeviceBlock> keep_tables, keep_bytes; // the lists may be released before the scorer runs
    };
    std::vector<ChildOffsets> child_off;
    double *d_ext = nullptr; // wide unions: the scorer's per-child tables in device memory (ScoreArgs::ext)
    UnionOrder *d_order = nullptr; // unions: the reference's aggregate child order per docId epoch
    // nested aggregates: child j (aggregate order) is itself an evaluated AND / OR (NULL: a leaf); its hits' positions inside it
    // are row j of d_hit_pos
    std::vector<std::shared_ptr<struct NestedSet>> nested;
    std::vector<uint8_t> child_tag; // RSResultData tag per child (aggregate order)
    size_t estimated = 0;           // num_estimated by the reference's rule: min over the children (AND), their sum (OR)
    // host-known bounds on the docIds the set can hold (lo_id > hi_id: none), filled by every constructor without a device read;
    // they bound the bitmap window of an OR over sets (II_UnionFilterBatchDevice)
    uint32_t lo_id = 0, hi_id = 0xFFFFFFFFu;
    std::unique_ptr<UnionOrder> h_order; // host copy of d_order (EXPLAINSCORE walks one hit's children in aggregate order)
    // a set of a device batch (II_IntersectBatchDevice, the filter batches): the hit count is known only on the device until
    // settle(); `ready` completes with the kernels that build the set
    bool pending = false;
    cudaEvent_t ready = nullptr;
    bool estimated_on_device = false; // a filter batch set whose num_estimated is summed on the device: d_len[1] until settle()
    // II_IntersectFilterBatchDevice with a child whose estimate is on the device: the child order waits for settle(), which sorts by
    // d_len[2 + i] (child i's num_estimated) times order_weight[i] (its sort weight; < 0 = a NOT child, sorted last); child_tag
    // is in the given order until then
    std::vector<double> order_weight;
    // completion events of the device filter batch calls that read this set as a child: the frees below wait for them
    std::vector<std::shared_ptr<struct SharedEvent>> readers;
    ~II_ResultSet() {
        if (ready) { // allocated on another stream, whose AND may still be writing: the frees below wait for it
            cudaStreamWaitEvent(ctx().stream, ready, 0);
            cudaEventDestroy(ready);
        }
        {
            std::lock_guard<std::mutex> g(readers_mu());
            for (const auto &r : readers) cudaStreamWaitEvent(ctx().stream, r->ev, 0);
        }
        dfree(d_docs);
        dfree(d_freqs);
        dfree(d_scores);
        dfree(d_len);
        dfree(d_hit_pos);
        dfree(d_slop);
        dfree(d_order);
        dfree(d_ext);
    }
};

// An evaluated AND / OR as ONE child of another aggregate — `(a|b) c`, the expansions of a stemmed term under an AND, a phrase
// inside a larger query.  The scorers recurse into it (src/ext/default.c:75-95,183-199,272-289,393-438: weight * sum / max over ITS
// children), the proximity checks and GetSlop merge its children's term positions (src/offset_vector.c:100-140,216-239).
struct NestedSet {
    std::unique_ptr<II_ResultSet> rs;
    std::vector<II_TermParams> terms; // of rs's children, in the order they were given to the constructor
    std::vector<std::string> term_strs; // their texts where known (EXPLAINSCORE of BM25STD prints them)
    double weight = 1.0;
    uint32_t *d_fsum = nullptr; // [rs->len] freq of the aggregate result = sum of its children's
    double *d_sub = nullptr;    // [rs->len] recursive score of every hit for the scorer being evaluated
    // merged term positions of every hit, re-encoded as varint deltas (built when a parent needs them)
    bool merged = false;
    uint8_t *d_mbytes = nullptr;
    uint32_t *d_moff_pos = nullptr, *d_moff_len = nullptr;
    ~NestedSet() {
        dfree(d_fsum);
        dfree(d_sub);
        dfree(d_mbytes);
        dfree(d_moff_pos);
        dfree(d_moff_len);
    }
};

// ------------------------------------------------------------------------------------------------
// host decoders (one block at a time; blocks are independent: the delta base restarts at first_doc_id)
// ------------------------------------------------------------------------------------------------
namespace {
// returns false on a malformed block (cursor ran past the buffer).  masks: the 32-bit field mask, or for the *Wide codecs
// whether the u128 mask meets (wf_lo, wf_hi) — same convention as the device decoder (mask_word in ii_kernels.cu)
bool decode_block(const II_BlockView &b, II_Codec codec, uint64_t wf_lo, uint64_t wf_hi, uint32_t *ids, uint32_t *freqs, uint32_t *masks) {
    const uint8_t *p = b.data, *end = b.data + b.len;
    uint64_t last = b.first_doc_id;
    for (uint32_t e = 0; e < b.num_entries; e++) {
        if (p >= end) return false;
        IIRecord r;
        p = ii_decode_record<true>(p, end, (int)codec, r);
        if (!p) return false;
        const uint64_t id = (codec == II_CODEC_RAW_DOCIDS_ONLY ? b.first_doc_id : last) + r.delta;
        if (id > 0xFFFFFFFEull) return false;
        last = id;
        ids[e] = (uint32_t)id;
        freqs[e] = r.freq;
        if (masks)
            masks[e] = ii_codec_is_wide((int)codec) ? (((r.mask_lo & wf_lo) | (r.mask_hi & wf_hi)) != 0 ? 1u : 0u) : (uint32_t)r.mask_lo;
    }
    return true;
}
} // namespace

static size_t from_blocks_batch(size_t n_lists, const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec, bool keep_offsets,
                                II_PostingList **out) {
    for (size_t i = 0; i < n_lists; i++) out[i] = nullptr;
    if ((int)codec < 0 || (int)codec >= kNumCodecs) return 0;
    keep_offsets = keep_offsets && ii_codec_has_offsets((int)codec);
    if (n_lists == 0) return 0;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return 0;
    size_t built = 0, first_list = 0;
    while (first_list < n_lists) {
        // sub-batch: < 4 GB of bytes and < 2^32 entries (32-bit tables)
        size_t stop = first_list, B = 0, nbytes = 0, n = 0;
        bool bad_ids = false;
        while (stop < n_lists) {
            size_t lb = 0, le = 0;
            for (size_t b = 0; b < nblocks[stop]; b++) {
                lb += blocks[stop][b].len;
                le += blocks[stop][b].num_entries;
                bad_ids |= blocks[stop][b].last_doc_id > 0xFFFFFFFEull;
            }
            if (stop > first_list && (nbytes + lb > ((size_t)3 << 30) || n + le > ((size_t)1 << 31))) break;
            nbytes += lb;
            n += le;
            B += nblocks[stop];
            stop++;
        }
        if (bad_ids || nbytes > ((size_t)4 << 30) - 64 || n >= ((size_t)1 << 32)) return built; // not representable on the device
        const size_t bytes_pad = (nbytes + 15 + 16) & ~(size_t)15; // the kernel copies whole 16-byte chunks
        const size_t stage_bytes = bytes_pad + (3 * B + 2) * 4;
        uint8_t *stg = c.stage(stage_bytes);
        if (!stg) return built;
        uint32_t *first = reinterpret_cast<uint32_t *>(stg + bytes_pad), *boff = first + B, *eoff = boff + B + 1;
        // tables (serial: cheap), then the byte gather on as many threads as the volume is worth
        std::vector<size_t> list_b0(stop - first_list + 1, 0), list_e0(stop - first_list + 1, 0);
        {
            size_t bi = 0, bo = 0, eo = 0;
            for (size_t l = first_list; l < stop; l++) {
                list_b0[l - first_list] = bi;
                list_e0[l - first_list] = eo;
                for (size_t b = 0; b < nblocks[l]; b++, bi++) {
                    first[bi] = (uint32_t)blocks[l][b].first_doc_id;
                    boff[bi] = (uint32_t)bo;
                    eoff[bi] = (uint32_t)eo;
                    bo += blocks[l][b].len;
                    eo += blocks[l][b].num_entries;
                }
            }
            boff[B] = (uint32_t)bo;
            eoff[B] = (uint32_t)eo;
            list_b0.back() = bi;
            list_e0.back() = eo;
        }
        const double tg = now_us();
        {
            const unsigned nt = std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 32u, (unsigned)(nbytes >> 22) + 1u}));
            auto work = [&](unsigned t) {
                const size_t l0 = first_list + (stop - first_list) * t / nt, l1 = first_list + (stop - first_list) * (t + 1) / nt;
                for (size_t l = l0; l < l1; l++) {
                    size_t bi = list_b0[l - first_list];
                    for (size_t b = 0; b < nblocks[l]; b++, bi++) memcpy(stg + boff[bi], blocks[l][b].data, blocks[l][b].len);
                }
            };
            if (nt == 1 || stop - first_list < 2 * (size_t)nt) {
                // few lists: split by blocks instead
                const unsigned nb_t = std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 32u, (unsigned)(nbytes >> 22) + 1u}));
                if (nb_t == 1) {
                    for (unsigned t = 0; t < nt; t++) work(t);
                } else {
                    std::vector<const II_BlockView *> flat(B);
                    size_t bi = 0;
                    for (size_t l = first_list; l < stop; l++)
                        for (size_t b = 0; b < nblocks[l]; b++) flat[bi++] = &blocks[l][b];
                    std::vector<std::thread> th;
                    for (unsigned t = 0; t < nb_t; t++)
                        th.emplace_back([&, t] {
                            for (size_t x = B * t / nb_t; x < B * (t + 1) / nb_t; x++) memcpy(stg + boff[x], flat[x]->data, flat[x]->len);
                        });
                    for (auto &x : th) x.join();
                }
            } else {
                std::vector<std::thread> th;
                for (unsigned t = 0; t < nt; t++) th.emplace_back(work, t);
                for (auto &x : th) x.join();
            }
            memset(stg + nbytes, 0, bytes_pad - nbytes);
        }
        c.stats.decode_host_us = now_us() - tg;
        const double t0 = now_us();
        auto blockmem = std::make_shared<SharedDeviceBlock>();
        blockmem->p = dalloc<uint8_t>((n ? n : 1) * (keep_offsets ? 16 : 8));
        uint8_t *d_stage = dalloc<uint8_t>(stage_bytes);
        bool ok = blockmem->p && d_stage;
        uint32_t *d_ids = reinterpret_cast<uint32_t *>(blockmem->p), *d_freqs = d_ids + n;
        uint32_t *d_off_pos = keep_offsets ? d_freqs + n : nullptr, *d_off_len = keep_offsets ? d_off_pos + n : nullptr;
        ok = ok && cudaMemcpyAsync(d_stage, stg, stage_bytes, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        const uint32_t *d_first = reinterpret_cast<const uint32_t *>(d_stage + bytes_pad), *d_boff = d_first + B, *d_eoff = d_boff + B + 1;
        ok = ok && ii_launch_decode_staged(d_stage, d_boff, d_first, d_eoff, (uint32_t)B, (int)codec, d_ids, d_freqs, nullptr, d_off_pos, d_off_len, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        c.stats.h2d_us = now_us() - t0;
        c.stats.kernel_launches += 1;
        std::shared_ptr<SharedDeviceBlock> bytesmem;
        if (keep_offsets && ok) {
            bytesmem = std::make_shared<SharedDeviceBlock>();
            bytesmem->p = d_stage;
        } else {
            dfree(d_stage);
        }
        if (!ok) {
            cudaGetLastError();
            return built;
        }
        for (size_t l = first_list; l < stop; l++) {
            auto *pl = new II_PostingList();
            const size_t e0 = list_e0[l - first_list], e1 = (l + 1 < stop) ? list_e0[l + 1 - first_list] : n;
            pl->owner = blockmem;
            pl->d_ids = d_ids + e0;
            pl->d_freqs = d_freqs + e0;
            if (keep_offsets) {
                pl->bytes_owner = bytesmem;
                pl->d_bytes = d_stage;
                pl->d_off_pos = d_off_pos + e0;
                pl->d_off_len = d_off_len + e0;
            }
            pl->n = pl->estimated = e1 - e0;
            pl->last_id = nblocks[l] ? (uint32_t)blocks[l][nblocks[l] - 1].last_doc_id : 0;
            pl->first_id = nblocks[l] ? (uint32_t)std::min<uint64_t>(blocks[l][0].first_doc_id, pl->last_id) : 0;
            out[l] = pl;
            built++;
        }
        first_list = stop;
    }
    return built;
}

extern "C" {

size_t II_PostingList_FromBlocksBatch(size_t n_lists, const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec,
                                      II_PostingList **out) {
    return from_blocks_batch(n_lists, blocks, nblocks, codec, false, out);
}
// same, keeping the term positions of a Full-codec index on the device (needed by slop / in-order intersections)
size_t II_PostingList_FromBlocksBatchOffsets(size_t n_lists, const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec,
                                             II_PostingList **out) {
    return from_blocks_batch(n_lists, blocks, nblocks, codec, true, out);
}
int II_PostingList_HasOffsets(const II_PostingList *pl) { return pl->d_off_len != nullptr; }

II_PostingList *II_PostingList_FromBlocks(const II_BlockView *blocks, size_t nblocks, II_Codec codec,
                                          uint32_t field_mask_filter, int decode_on_device) {
    const uint64_t wide[2] = {field_mask_filter, 0};
    return II_PostingList_FromBlocksWideMask(blocks, nblocks, codec, wide, decode_on_device);
}
II_PostingList *II_PostingList_FromBlocksWideMask(const II_BlockView *blocks, size_t nblocks, II_Codec codec, const uint64_t filter128[2],
                                                  int decode_on_device) {
    if ((int)codec < 0 || (int)codec >= kNumCodecs) return nullptr;
    const uint64_t wf_lo = filter128 ? filter128[0] : 0, wf_hi = filter128 ? filter128[1] : 0;
    const bool wide = ii_codec_is_wide((int)codec);
    if (!wide && (wf_hi != 0 || wf_lo > 0xFFFFFFFFull)) return nullptr; // a 32-bit mask codec cannot meet bits above 31: ask the wide codec
    // what the ordered compaction tests: the 32-bit mask itself, or the decoder's "meets the u128 filter" flag
    const uint32_t field_mask_filter = wide ? ((wf_lo | wf_hi) ? 1u : 0u) : (uint32_t)wf_lo;
    if (decode_on_device && field_mask_filter == 0) { // the common case rides the batch decoder (one copy, one launch, one sync)
        II_PostingList *one = nullptr;
        const II_BlockView *bl[1] = {blocks};
        const size_t nb[1] = {nblocks};
        II_PostingList_FromBlocksBatch(1, bl, nb, codec, &one);
        return one;
    }
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    std::vector<uint32_t> entry_off(nblocks + 1, 0);
    std::vector<uint64_t> byte_off(nblocks + 1, 0);
    for (size_t b = 0; b < nblocks; b++) {
        entry_off[b + 1] = entry_off[b] + blocks[b].num_entries;
        byte_off[b + 1] = byte_off[b] + blocks[b].len;
        if (blocks[b].last_doc_id > 0xFFFFFFFEull) return nullptr;
    }
    const size_t n = entry_off[nblocks];
    auto *pl = new II_PostingList();
    pl->estimated = n;
    const bool need_mask = field_mask_filter != 0 && ii_codec_has_mask((int)codec);
    uint32_t *d_ids = dalloc<uint32_t>(n), *d_freqs = dalloc<uint32_t>(n), *d_masks = need_mask ? dalloc<uint32_t>(n) : nullptr;
    bool ok = d_ids && d_freqs && (!need_mask || d_masks);
    if (ok && n) {
        if (decode_on_device) {
            // ship the raw block bytes (gathered into pinned staging by all cores), decode with one thread per block
            const size_t nbytes = byte_off[nblocks];
            uint8_t *stg = c.stage(nbytes + nblocks * 8 + 16);
            if (!stg) {
                dfree(d_ids);
                dfree(d_freqs);
                dfree(d_masks);
                delete pl;
                return nullptr;
            }
            uint8_t *bytes = stg;
            uint64_t *first = reinterpret_cast<uint64_t *>(stg + ((nbytes + 7) & ~(size_t)7));
            const double tg = now_us();
            {
                unsigned nt = std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 32u, (unsigned)(nblocks / 4096 + 1)}));
                std::vector<std::thread> th;
                for (unsigned t = 0; t < nt; t++)
                    th.emplace_back([&, t] {
                        const size_t b0 = nblocks * t / nt, b1 = nblocks * (t + 1) / nt;
                        for (size_t b = b0; b < b1; b++) {
                            memcpy(bytes + byte_off[b], blocks[b].data, blocks[b].len);
                            first[b] = blocks[b].first_doc_id;
                        }
                    });
                for (auto &x : th) x.join();
            }
            c.stats.decode_host_us = now_us() - tg; // host share of the device-decode route: the gather
            uint8_t *d_bytes = dalloc<uint8_t>(nbytes + 8);
            uint64_t *d_boff = dalloc<uint64_t>(nblocks + 1), *d_first = dalloc<uint64_t>(nblocks);
            uint32_t *d_eoff = dalloc<uint32_t>(nblocks + 1);
            ok = d_bytes && d_boff && d_first && d_eoff;
            const double t0 = now_us();
            ok = ok && cudaMemcpyAsync(d_bytes, bytes, nbytes, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(d_boff, byte_off.data(), (nblocks + 1) * 8, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(d_first, first, nblocks * 8, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(d_eoff, entry_off.data(), (nblocks + 1) * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
            ok = ok && ii_launch_decode(d_bytes, d_boff, d_first, d_eoff, (uint32_t)nblocks, (int)codec, wf_lo, wf_hi, d_ids, d_freqs, d_masks,
                                        c.stream) == cudaSuccess;
            ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
            c.stats.h2d_us = now_us() - t0;
            c.stats.kernel_launches += 1;
            dfree(d_bytes);
            dfree(d_boff);
            dfree(d_first);
            dfree(d_eoff);
        } else {
            uint8_t *stg = c.stage(n * 4 * (need_mask ? 3 : 2));
            uint32_t *h_ids = reinterpret_cast<uint32_t *>(stg), *h_freqs = h_ids + n, *h_masks = need_mask ? h_freqs + n : nullptr;
            ok = stg != nullptr;
            if (ok) {
                const double t0 = now_us();
                unsigned nt = std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 64u, (unsigned)(nblocks / 256 + 1)}));
                std::vector<std::thread> th;
                std::vector<char> good(nt, 1);
                for (unsigned t = 0; t < nt; t++)
                    th.emplace_back([&, t] {
                        for (size_t b = t; b < nblocks; b += nt)
                            if (!decode_block(blocks[b], codec, wf_lo, wf_hi, h_ids + entry_off[b], h_freqs + entry_off[b],
                                              h_masks ? h_masks + entry_off[b] : nullptr))
                                good[t] = 0;
                    });
                for (auto &x : th) x.join();
                for (char gd : good) ok = ok && gd;
                c.stats.decode_host_us = now_us() - t0;
                const double t1 = now_us();
                ok = ok && cudaMemcpyAsync(d_ids, h_ids, n * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
                ok = ok && cudaMemcpyAsync(d_freqs, h_freqs, n * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
                if (need_mask) ok = ok && cudaMemcpyAsync(d_masks, h_masks, n * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
                ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
                c.stats.h2d_us = now_us() - t1;
            }
        }
    }
    size_t kept = n;
    if (ok && need_mask && n) { // FilterMaskReader: drop records whose mask misses the filter, order kept
        const uint32_t chunks = (uint32_t)((n + 1023) / 1024);
        uint32_t *d_counts = dalloc<uint32_t>(chunks), *d_offs = dalloc<uint32_t>(chunks);
        uint32_t *d_ids2 = dalloc<uint32_t>(n), *d_freqs2 = dalloc<uint32_t>(n);
        ok = d_counts && d_offs && d_ids2 && d_freqs2;
        ok = ok && ii_launch_mask_filter(d_ids, d_freqs, d_masks, (uint32_t)n, field_mask_filter, d_counts, d_offs, c.d_total,
                                         d_ids2, d_freqs2, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(c.h_total, c.d_total, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        c.stats.kernel_launches += 3;
        if (ok) {
            kept = *c.h_total;
            std::swap(d_ids, d_ids2);
            std::swap(d_freqs, d_freqs2);
        }
        dfree(d_ids2);
        dfree(d_freqs2);
        dfree(d_counts);
        dfree(d_offs);
    }
    dfree(d_masks);
    if (!ok) {
        dfree(d_ids);
        dfree(d_freqs);
        delete pl;
        return nullptr;
    }
    pl->d_ids = d_ids;
    pl->d_freqs = d_freqs;
    pl->n = kept;
    if (kept) copy_sync(&pl->last_id, d_ids + kept - 1, 4, cudaMemcpyDeviceToHost);
    if (kept && nblocks) pl->first_id = (uint32_t)std::min<uint64_t>(blocks[0].first_doc_id, pl->last_id);
    return pl;
}

II_PostingList *II_PostingList_FromArrays(const uint64_t *doc_ids, const uint32_t *freqs, size_t n) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    std::vector<uint32_t> ids32(n), f32(n, 1);
    for (size_t i = 0; i < n; i++) {
        if (doc_ids[i] > 0xFFFFFFFEull || (i && doc_ids[i] <= doc_ids[i - 1])) return nullptr;
        ids32[i] = (uint32_t)doc_ids[i];
        if (freqs) f32[i] = freqs[i];
    }
    auto *pl = new II_PostingList();
    pl->d_ids = dalloc<uint32_t>(n);
    pl->d_freqs = dalloc<uint32_t>(n);
    if (!pl->d_ids || !pl->d_freqs ||
        (n && (copy_sync(pl->d_ids, ids32.data(), n * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
               copy_sync(pl->d_freqs, f32.data(), n * 4, cudaMemcpyHostToDevice) != cudaSuccess))) {
        delete pl;
        return nullptr;
    }
    pl->n = pl->estimated = n;
    pl->last_id = n ? ids32[n - 1] : 0;
    pl->first_id = n ? ids32[0] : 0;
    return pl;
}

II_PostingList *II_PostingList_FromDevice(const uint32_t *d_doc_ids, const uint32_t *d_freqs, size_t n) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    auto *pl = new II_PostingList();
    pl->d_ids = dalloc<uint32_t>(n);
    pl->d_freqs = dalloc<uint32_t>(n);
    bool ok = pl->d_ids && pl->d_freqs;
    if (ok && n) {
        ok = copy_sync(pl->d_ids, d_doc_ids, n * 4, cudaMemcpyDeviceToDevice) == cudaSuccess;
        if (d_freqs)
            ok = ok && copy_sync(pl->d_freqs, d_freqs, n * 4, cudaMemcpyDeviceToDevice) == cudaSuccess;
        else {
            std::vector<uint32_t> ones(n, 1);
            ok = ok && copy_sync(pl->d_freqs, ones.data(), n * 4, cudaMemcpyHostToDevice) == cudaSuccess;
        }
        ok = ok && copy_sync(&pl->last_id, pl->d_ids + n - 1, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    if (!ok) {
        delete pl;
        return nullptr;
    }
    pl->n = pl->estimated = n;
    return pl;
}

// ---- the index WRITER: InvertedIndex::add_record (RS/inverted_index/src/index/core.rs:235-358) for every term codec and the
// numeric one — the ingest side of posting storage: the IndexBlocks it produces are byte-identical to the reference's
// (tests/test_index_writer.py against the oracle restatement and the reference's golden vectors), so a host can keep its postings
// in this library's blocks and hand them to the decoders above without an encoding of its own.
struct II_IndexWriter {
    struct Block {
        uint64_t first = 0, last = 0;
        uint16_t n = 0;
        std::vector<uint8_t> buf;
    };
    int codec = 0; // 0..12 term codecs, 13 numeric
    bool compress_floats = false;
    std::vector<Block> blocks;
    size_t unique_docs = 0;
    bool multi_value = false;
    uint16_t per_block() const { return (codec == II_CODEC_DOCIDS_ONLY || codec == II_CODEC_RAW_DOCIDS_ONLY) ? 1000 : 100; } // codec/mod.rs:69
};
static size_t writer_add(II_IndexWriter *w, uint64_t doc_id, const std::function<size_t(uint64_t delta, uint8_t *out)> &encode, uint64_t max_delta,
                         bool allow_duplicates, size_t reserve) {
    const bool have_last = !w->blocks.empty();
    const bool same_doc = have_last && w->blocks.back().last == doc_id;
    if (same_doc && !allow_duplicates) return 0; // :244-256: a repeated docId carries nothing new for these codecs
    if (have_last && doc_id < w->blocks.back().last) return 0; // documents arrive in docId order
    // take_block :339-358: a full block is only left for a NEW document (the records of one document stay together)
    if (!have_last || (!same_doc && w->blocks.back().n >= w->per_block())) {
        w->blocks.emplace_back();
        w->blocks.back().first = w->blocks.back().last = doc_id;
    }
    II_IndexWriter::Block *b = &w->blocks.back();
    const uint64_t base = (w->codec == II_CODEC_RAW_DOCIDS_ONLY) ? b->first : b->last; // raw_doc_ids_only.rs:40-47
    uint64_t delta = doc_id - base;
    if (delta > max_delta) { // :272-285: the delta does not fit this encoder: a fresh block, delta 0
        w->blocks.emplace_back();
        b = &w->blocks.back();
        b->first = b->last = doc_id;
        delta = 0;
    }
    const size_t before = b->buf.size();
    b->buf.resize(before + reserve);
    const size_t n = encode(delta, b->buf.data() + before);
    b->buf.resize(before + n);
    b->n++;
    b->last = doc_id;
    if (same_doc)
        w->multi_value = true;
    else
        w->unique_docs++;
    return n;
}
II_IndexWriter *II_IndexWriter_New(II_Codec codec) {
    if ((int)codec < 0 || (int)codec >= kNumCodecs) return nullptr;
    auto *w = new II_IndexWriter();
    w->codec = (int)codec;
    return w;
}
II_IndexWriter *II_IndexWriter_NewNumeric(int compress_floats) {
    auto *w = new II_IndexWriter();
    w->codec = 13;
    w->compress_floats = compress_floats != 0;
    return w;
}
void II_IndexWriter_Free(II_IndexWriter *w) { delete w; }
size_t II_IndexWriter_Add(II_IndexWriter *w, uint64_t doc_id, uint32_t freq, uint64_t mask_lo, uint64_t mask_hi, const uint8_t *offsets,
                          uint32_t offsets_len) {
    if (!w || w->codec > 12) return 0;
    if (!ii_codec_has_offsets(w->codec)) offsets_len = 0;
    return writer_add(
        w, doc_id,
        [&](uint64_t delta, uint8_t *out) { return ii_encode_record(w->codec, (uint32_t)delta, freq, mask_lo, mask_hi, offsets, offsets_len, out); },
        0xFFFFFFFFull, false, 64 + (size_t)offsets_len);
}
size_t II_IndexWriter_AddNumeric(II_IndexWriter *w, uint64_t doc_id, double value) {
    if (!w || w->codec != 13) return 0;
    return writer_add(
        w, doc_id, [&](uint64_t delta, uint8_t *out) { return ii_encode_numeric(delta, value, w->compress_floats, out); },
        ((uint64_t)1 << 56) - 1 /* NumericDelta: 7 bytes, numeric.rs:297-305 */, true /* ALLOW_DUPLICATES :323 */, 24);
}
size_t II_IndexWriter_NumBlocks(const II_IndexWriter *w) { return w->blocks.size(); }
size_t II_IndexWriter_NumDocs(const II_IndexWriter *w) { return w->unique_docs; }
int II_IndexWriter_Block(const II_IndexWriter *w, size_t i, II_BlockView *out) {
    if (!w || i >= w->blocks.size() || !out) return -1;
    const auto &b = w->blocks[i];
    *out = II_BlockView{b.first, b.last, b.n, b.buf.data(), b.buf.size()};
    return 0;
}

// ---- numeric index blocks (RS/inverted_index/src/codec/numeric.rs) -> device (docId, value) arrays; range filters over them
struct II_NumericList {
    uint32_t *d_ids = nullptr;
    double *d_values = nullptr;
    size_t n = 0;
    uint32_t first_id = 0, last_id = 0; // the blocks' docId bounds
    ~II_NumericList() {
        dfree(d_ids);
        dfree(d_values);
    }
};
II_NumericList *II_NumericList_FromBlocks(const II_BlockView *blocks, size_t nblocks) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    std::vector<uint32_t> entry_off(nblocks + 1, 0);
    std::vector<uint64_t> byte_off(nblocks + 1, 0), first(nblocks, 0);
    for (size_t b = 0; b < nblocks; b++) {
        entry_off[b + 1] = entry_off[b] + blocks[b].num_entries;
        byte_off[b + 1] = byte_off[b] + blocks[b].len;
        first[b] = blocks[b].first_doc_id;
        if (blocks[b].last_doc_id > 0xFFFFFFFEull) return nullptr;
        // validate on the host what the device decoder trusts: every record stays inside its block
        const uint8_t *p = blocks[b].data, *end = p + blocks[b].len;
        for (uint32_t e = 0; e < blocks[b].num_entries; e++) {
            uint64_t d;
            double v;
            p = ii_decode_numeric<true>(p, end, d, v);
            if (!p) return nullptr;
        }
    }
    const size_t n = entry_off[nblocks], nbytes = byte_off[nblocks];
    auto *nl = new II_NumericList();
    nl->n = n;
    if (nblocks) {
        nl->last_id = (uint32_t)blocks[nblocks - 1].last_doc_id;
        nl->first_id = (uint32_t)std::min<uint64_t>(blocks[0].first_doc_id, nl->last_id);
    }
    nl->d_ids = dalloc<uint32_t>(n ? n : 1);
    nl->d_values = dalloc<double>(n ? n : 1);
    uint8_t *stg = c.stage(nbytes + 16);
    uint8_t *d_bytes = dalloc<uint8_t>(nbytes + 16);
    uint64_t *d_boff = dalloc<uint64_t>(nblocks + 1), *d_first = dalloc<uint64_t>(nblocks + 1);
    uint32_t *d_eoff = dalloc<uint32_t>(nblocks + 1);
    bool ok = nl->d_ids && nl->d_values && stg && d_bytes && d_boff && d_first && d_eoff;
    if (ok && n) {
        for (size_t b = 0; b < nblocks; b++) memcpy(stg + byte_off[b], blocks[b].data, blocks[b].len);
        ok = cudaMemcpyAsync(d_bytes, stg, nbytes, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(d_boff, byte_off.data(), (nblocks + 1) * 8, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(d_first, first.data(), nblocks * 8, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(d_eoff, entry_off.data(), (nblocks + 1) * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        ok = ok && ii_launch_decode_numeric(d_bytes, d_boff, d_first, d_eoff, (uint32_t)nblocks, nl->d_ids, nl->d_values, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        c.stats.kernel_launches += 1;
    }
    dfree(d_bytes);
    dfree(d_boff);
    dfree(d_first);
    dfree(d_eoff);
    if (!ok) {
        delete nl;
        return nullptr;
    }
    return nl;
}
size_t II_NumericList_Len(const II_NumericList *nl) { return nl->n; }
void II_NumericList_Free(II_NumericList *nl) { delete nl; }
int II_NumericList_Fetch(const II_NumericList *nl, uint64_t *doc_ids, double *values) {
    if (!nl->n) return 0;
    std::vector<uint32_t> ids(nl->n);
    bool ok = copy_sync(ids.data(), nl->d_ids, nl->n * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    if (values) ok = ok && copy_sync(values, nl->d_values, nl->n * 8, cudaMemcpyDeviceToHost) == cudaSuccess;
    if (doc_ids)
        for (size_t i = 0; i < nl->n; i++) doc_ids[i] = ids[i];
    return ok ? 0 : -1;
}
// FilterNumericReader (reader/numeric.rs:80-170) + one result per document (the numeric iterator skips the further records of a
// multi-value document): ascending docIds, freq 1.  The list is a term-like leaf for AND / OR / hybrid pre-filters.
II_PostingList *II_NumericList_Filter(const II_NumericList *nl, double min, double max, int min_inclusive, int max_inclusive) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init() || !nl) return nullptr;
    const size_t n = nl->n;
    auto *pl = new II_PostingList();
    pl->d_ids = dalloc<uint32_t>(n ? n : 1);
    pl->d_freqs = dalloc<uint32_t>(n ? n : 1);
    const uint32_t chunks = (uint32_t)((n + 1023) / 1024);
    uint32_t *d_counts = dalloc<uint32_t>(chunks ? chunks : 1), *d_offs = dalloc<uint32_t>(chunks ? chunks : 1);
    bool ok = pl->d_ids && pl->d_freqs && d_counts && d_offs;
    size_t kept = 0;
    if (ok && n) {
        ok = ii_launch_numeric_filter(nl->d_ids, nl->d_values, (uint32_t)n, min, max, min_inclusive != 0, max_inclusive != 0, d_counts, d_offs,
                                      c.d_total, pl->d_ids, pl->d_freqs, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(c.h_total, c.d_total, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        c.stats.kernel_launches += 3;
        if (ok) kept = *c.h_total;
        if (ok && kept) ok = copy_sync(&pl->last_id, pl->d_ids + kept - 1, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    dfree(d_counts);
    dfree(d_offs);
    if (!ok) {
        delete pl;
        return nullptr;
    }
    pl->n = pl->estimated = kept;
    pl->first_id = kept ? std::min(nl->first_id, pl->last_id) : 0;
    pl->result_tag = 16; // numeric results
    return pl;
}

// every docId 1..top_id with freq 1 (what a wildcard child contributes to an aggregate)
static II_PostingList *posting_list_all_docs(uint64_t top_id) {
    if (top_id > 0xFFFFFFFEull) return nullptr;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    auto *pl = new II_PostingList();
    const size_t n = (size_t)top_id;
    pl->d_ids = dalloc<uint32_t>(n ? n : 1);
    pl->d_freqs = dalloc<uint32_t>(n ? n : 1);
    bool ok = pl->d_ids && pl->d_freqs;
    ok = ok && ii_launch_iota(pl->d_ids, pl->d_freqs, (uint32_t)n, c.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    if (!ok) {
        delete pl;
        return nullptr;
    }
    pl->n = pl->estimated = n;
    pl->last_id = (uint32_t)top_id;
    pl->result_tag = 8; // virtual results
    return pl;
}

size_t II_PostingList_Len(const II_PostingList *pl) { return pl->n; }
size_t II_PostingList_NumEstimated(const II_PostingList *pl) { return pl->estimated; }
void II_PostingList_Free(II_PostingList *pl) { delete pl; }

// ------------------------------------------------------------------------------------------------
static II_DocTable *doctable_from(size_t max_doc_id, const uint32_t *len, const float *score, const uint32_t *maxf,
                                  cudaMemcpyKind kind) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    auto *dt = new II_DocTable();
    dt->max_doc = max_doc_id;
    const size_t n = max_doc_id + 1;
    bool ok = true;
    if (len) {
        dt->d_len = dalloc<uint32_t>(n);
        ok = ok && dt->d_len && copy_sync(dt->d_len, len, n * 4, kind) == cudaSuccess;
    }
    if (score) {
        dt->d_score = dalloc<float>(n);
        ok = ok && dt->d_score && copy_sync(dt->d_score, score, n * 4, kind) == cudaSuccess;
    }
    if (maxf) {
        dt->d_maxf = dalloc<uint32_t>(n);
        ok = ok && dt->d_maxf && copy_sync(dt->d_maxf, maxf, n * 4, kind) == cudaSuccess;
    }
    if (!ok) {
        delete dt;
        return nullptr;
    }
    return dt;
}
II_DocTable *II_DocTable_New(size_t max_doc_id, const uint32_t *doc_len, const float *doc_score, const uint32_t *max_term_freq) {
    return doctable_from(max_doc_id, doc_len, doc_score, max_term_freq, cudaMemcpyHostToDevice);
}
II_DocTable *II_DocTable_FromDevice(size_t max_doc_id, const uint32_t *d_doc_len, const float *d_doc_score,
                                    const uint32_t *d_max_term_freq) {
    return doctable_from(max_doc_id, d_doc_len, d_doc_score, d_max_term_freq, cudaMemcpyDeviceToDevice);
}
void II_DocTable_Free(II_DocTable *dt) { delete dt; }
int II_DocTable_SetPayloads(II_DocTable *dt, const uint8_t *payloads, const uint64_t *offsets) {
    if (!dt || !offsets) return -1;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return -1;
    const size_t n = dt->max_doc + 2, bytes = offsets[dt->max_doc + 1];
    for (size_t d = 0; d + 1 < n; d++)
        if (offsets[d] > offsets[d + 1]) return -1;
    dfree(dt->d_payloads);
    dfree(dt->d_payload_off);
    dt->d_payloads = dalloc<uint8_t>(bytes ? bytes : 1);
    dt->d_payload_off = dalloc<uint64_t>(n);
    bool ok = dt->d_payloads && dt->d_payload_off;
    ok = ok && copy_sync(dt->d_payload_off, offsets, n * 8, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && (!bytes || (payloads && copy_sync(dt->d_payloads, payloads, bytes, cudaMemcpyHostToDevice) == cudaSuccess));
    if (!ok) {
        dfree(dt->d_payloads);
        dfree(dt->d_payload_off);
        dt->d_payloads = nullptr;
        dt->d_payload_off = nullptr;
        return -1;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// AND / OR: enqueue-only cores (no host synchronisation) + synchronous public wrappers
// ------------------------------------------------------------------------------------------------
namespace {

// The shape every aggregate starts from: n children in the given order, each tagged `tag` (RSResultData), none nested, no term
// positions
void init_children(II_ResultSet *rs, size_t n, uint8_t tag) {
    rs->n_children = (uint32_t)n;
    rs->child_order.resize(n);
    for (size_t i = 0; i < n; i++) rs->child_order[i] = (uint32_t)i;
    rs->child_off.assign(n, II_ResultSet::ChildOffsets());
    rs->nested.assign(n, nullptr);
    rs->child_tag.assign(n, tag);
}

// sort key of Intersection::new_with_slop_order (intersection.rs:110-120): num_estimated * intersection_sort_weight, as doubles;
// NOT / OPTIONAL children estimate max_doc_id (not.rs / optional.rs num_estimated): they sort behind every other child
inline double and_sort_key(bool required, double estimated, double sort_weight) { return required ? estimated * sort_weight : 0x1p62; }
struct AndKey {
    bool required;
    double estimated, sort_weight;
};
// Intersection::new's aggregate child order (intersection.rs:110-145): a stable sort of the n children ascending by and_sort_key of
// key(i), so NOT / OPTIONAL children come last in their given order.  rs->child_order becomes that order, and rs->child_tag, given
// in the children's given order, is permuted into it.
extern "C++" template <class Key> void and_order(II_ResultSet *rs, size_t n, Key &&key) {
    std::vector<double> k(n);
    for (size_t i = 0; i < n; i++) {
        const AndKey a = key(i);
        k[i] = and_sort_key(a.required, a.estimated, a.sort_weight);
    }
    std::vector<uint32_t> order(n);
    for (size_t i = 0; i < n; i++) order[i] = (uint32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return k[a] < k[b]; });
    std::vector<uint8_t> tag(n);
    for (size_t j = 0; j < n; j++) tag[j] = rs->child_tag[order[j]];
    rs->child_order = std::move(order);
    rs->child_tag = std::move(tag);
}

struct PhraseSpec {
    uint32_t max_slop; // 0xFFFFFFFF: no limit (in-order only)
    bool in_order;
};
// Enqueue the kernels of an intersection on ctx().stream.  On return rs->d_len holds (will hold, in
// stream order) the number of hits; rs->len is NOT set.  *trivially_empty = an input list is empty.
// modes (nullable): per list 0 = required, 1 = NOT, 2 = OPTIONAL (IntersectArgs::mode); at least one list is required
bool intersect_enqueue(Ctx &c, II_PostingList *const *lists, size_t n, II_ResultSet *rs, bool *trivially_empty, const int *modes = nullptr,
                       const PhraseSpec *phrase = nullptr) {
    auto mode_of = [&](size_t i) { return modes ? modes[i] : 0; };
    if (phrase && n > (size_t)kPhraseMaxLists) return false;
    init_children(rs, n, 4);
    for (size_t i = 0; i < n; i++) rs->child_tag[i] = mode_of(i) == 1 ? 8 : lists[i]->result_tag;
    // an in-order intersection keeps the children as given: their order is the order the terms must appear in
    // (intersection.rs new_sorted_by: `if !in_order { children.sort_by(compare) }`)
    if (!(phrase && phrase->in_order))
        and_order(rs, n, [&](size_t i) { return AndKey{mode_of(i) == 0, (double)lists[i]->estimated, lists[i]->sort_weight}; });
    const std::vector<uint32_t> &order = rs->child_order;
    // the kernel is driven by the REQUIRED list with the fewest actual entries (a field-mask filter may make
    // that differ from the estimate order); the aggregate child order stays the reference's
    size_t drv = n;
    for (size_t i = 0; i < n; i++)
        if (mode_of(order[i]) == 0 && (drv == n || lists[order[i]]->n < lists[order[drv]]->n)) drv = i;
    if (drv == n) return false;
    bool any_nested = false;
    rs->estimated = (size_t)-1;
    for (size_t j = 0; j < n; j++) {
        const II_PostingList *L = lists[order[j]];
        if (mode_of(order[j]) == 0) {
            rs->estimated = std::min(rs->estimated, L->estimated); // NOT / OPTIONAL estimate max_doc_id
            rs->lo_id = std::max(rs->lo_id, L->first_id);          // every hit is in each required list
            rs->hi_id = std::min(rs->hi_id, L->last_id);
        }
        if (L->nested && mode_of(order[j]) != 1) {
            rs->nested[j] = L->nested;
            any_nested = true;
        }
    }
    *trivially_empty = false;
    for (size_t i = 0; i < n; i++) *trivially_empty |= mode_of(i) == 0 && lists[i]->n == 0;
    if (*trivially_empty) return true;
    const II_PostingList *A = lists[order[drv]];
    const uint32_t nchunks = (uint32_t)((A->n + kIIChunk - 1) / kIIChunk);
    const size_t stride = (size_t)nchunks * kIIChunk;
    rs->cap = A->n;
    rs->d_docs = dalloc<uint32_t>(rs->cap);
    rs->d_freqs = dalloc<uint32_t>(rs->cap * n);
    rs->d_scores = dalloc<double>(rs->cap);
    rs->d_len = dalloc<uint32_t>(4);
    uint32_t *tmp_idx = dalloc<uint32_t>(stride), *tmp_pos = dalloc<uint32_t>(stride * n);
    uint32_t *counts = dalloc<uint32_t>(nchunks), *offsets = dalloc<uint32_t>(nchunks);
    const bool check_phrase = phrase && n > 1;
    // keep the hits' posting positions when a child carries term positions: GetSlop needs them later (II_Score)
    bool keep_pos = false;
    for (size_t i = 0; i < n && n > 1; i++) keep_pos |= mode_of(i) != 1 && lists[i]->d_off_len != nullptr;
    keep_pos |= any_nested; // the scorers reach a nested child's recursive value through the hit's position inside it
    if (keep_pos) rs->d_hit_pos = dalloc<uint32_t>(rs->cap * n);
    const uint32_t pchunks = (uint32_t)((rs->cap + 1023) / 1024);
    // phrase path: the gather fills scratch rows, the filter compacts the survivors into the result set
    uint32_t *pre_freqs = check_phrase ? dalloc<uint32_t>(rs->cap * n) : nullptr, *pre_pos = check_phrase ? dalloc<uint32_t>(rs->cap * n) : nullptr;
    uint32_t *flags = check_phrase ? dalloc<uint32_t>(rs->cap) : nullptr;
    uint32_t *pcounts = check_phrase ? dalloc<uint32_t>(pchunks) : nullptr, *poffsets = check_phrase ? dalloc<uint32_t>(pchunks) : nullptr;
    uint32_t *pre_docs = check_phrase ? dalloc<uint32_t>(rs->cap) : nullptr, *pre_len = check_phrase ? dalloc<uint32_t>(4) : nullptr;
    bool ok = rs->d_docs && rs->d_freqs && rs->d_scores && rs->d_len && tmp_idx && tmp_pos && counts && offsets && (!keep_pos || rs->d_hit_pos) &&
              (!check_phrase || (pre_freqs && pre_pos && flags && pcounts && poffsets && pre_docs && pre_len));
    if (ok) {
        // kernel list order: driver first, then the rest ascending by length (cheap rejections first)
        std::vector<uint32_t> korder;
        korder.push_back((uint32_t)drv);
        std::vector<uint32_t> rest;
        for (size_t i = 0; i < n; i++)
            if (i != drv) rest.push_back((uint32_t)i);
        std::stable_sort(rest.begin(), rest.end(), [&](uint32_t x, uint32_t y) { return lists[order[x]]->n < lists[order[y]]->n; });
        korder.insert(korder.end(), rest.begin(), rest.end());
        IntersectArgs a{};
        a.n = (uint32_t)n;
        for (size_t i = 0; i < n; i++) {
            a.ids[i] = lists[order[korder[i]]]->d_ids;
            a.len[i] = (uint32_t)lists[order[korder[i]]]->n;
            a.mode[i] = (uint8_t)mode_of(order[korder[i]]);
        }
        a.tmp_idx = tmp_idx;
        a.tmp_pos = tmp_pos;
        a.counts = counts;
        a.stride = stride;
        cudaEventRecord(c.e0, c.stream);
        ok = ii_launch_intersect(a, nchunks, offsets, check_phrase ? pre_len : rs->d_len, c.stream) == cudaSuccess;
        GatherArgs ga{};
        ga.ids0 = A->d_ids;
        ga.n = (uint32_t)n;
        ga.tmp_idx = tmp_idx;
        ga.tmp_pos = tmp_pos;
        ga.counts = counts;
        ga.offsets = offsets;
        ga.stride = stride;
        ga.fstride = rs->cap;
        for (size_t k = 0; k < n; k++) {
            ga.freqs[k] = lists[order[korder[k]]]->d_freqs;
            ga.mode[k] = (uint8_t)mode_of(order[korder[k]]);
            ga.row[k] = (uint8_t)korder[k]; // kernel slot k holds aggregate child korder[k]
        }
        // rows land at their aggregate child index
        ga.out_doc = check_phrase ? pre_docs : rs->d_docs;
        ga.out_freq = check_phrase ? pre_freqs : rs->d_freqs;
        ga.out_pos = check_phrase ? pre_pos : rs->d_hit_pos;
        ok = ok && ii_launch_gather(ga, nchunks, c.stream) == cudaSuccess;
        for (size_t j = 0; j < n && keep_pos; j++) { // aggregate child j
            const II_PostingList *L = lists[order[j]];
            II_ResultSet::ChildOffsets &co = rs->child_off[j];
            if (mode_of(order[j]) == 1 || !L->d_off_len) continue;
            co.bytes = L->d_bytes;
            co.off_pos = L->d_off_pos;
            co.off_len = L->d_off_len;
            co.keep_tables = L->owner;
            co.keep_bytes = L->bytes_owner;
        }
        if (ok && check_phrase) {
            // slop / in-order: one thread per hit walks the term positions of its children (kept on the device by the
            // decoder), survivors are compacted in order straight into the aggregate rows
            PhraseArgs pa{};
            pa.n = (uint32_t)n;
            pa.max_slop = phrase->max_slop;
            pa.in_order = phrase->in_order ? 1 : 0;
            pa.pos = pre_pos;
            pa.fstride = rs->cap;
            for (size_t j = 0; j < n; j++) {
                const II_PostingList *L = lists[order[j]];
                pa.bytes[j] = L->d_bytes;
                pa.off_pos[j] = L->d_off_pos;
                pa.off_len[j] = mode_of(order[j]) == 1 ? nullptr : L->d_off_len;
            }
            ok = ii_launch_phrase_filter(pa, pre_len, (uint32_t)rs->cap, flags, pcounts, poffsets, rs->d_len, pre_docs, pre_freqs, rs->cap,
                                         rs->d_docs, rs->d_freqs, rs->d_hit_pos, rs->cap, c.stream) == cudaSuccess;
            c.stats.kernel_launches += 4;
        }
        cudaEventRecord(c.e1, c.stream);
        c.stats.kernel_launches += 3;
    }
    dfree(pre_freqs);
    dfree(pre_pos);
    dfree(flags);
    dfree(pcounts);
    dfree(poffsets);
    dfree(pre_docs);
    dfree(pre_len);
    dfree(tmp_idx);
    dfree(tmp_pos);
    dfree(counts);
    dfree(offsets);
    return ok;
}

// Merged term positions of a nested set's hits (MergeOffsetsArgs): its own nested children first, then two passes over its hits.
// One host synchronisation (the size of the byte buffer).
bool ensure_merged(Ctx &c, NestedSet *ns) {
    if (ns->merged) return true;
    II_ResultSet *rs = ns->rs.get();
    const size_t m = rs->len;
    if (rs->n_children > (uint32_t)kIIMaxLists) return false;
    if (!rs->has_freqs && !rs->d_hit_pos) return false; // a quick union does not know which children matched
    MergeOffsetsArgs a{};
    a.n = rs->n_children;
    a.is_union = rs->is_union ? 1 : 0;
    a.pos = rs->d_hit_pos;
    a.freqs = rs->d_freqs;
    a.fstride = rs->cap;
    for (uint32_t j = 0; j < rs->n_children; j++) {
        if (j < rs->nested.size() && rs->nested[j]) {
            NestedSet *ch = rs->nested[j].get();
            if (!ensure_merged(c, ch)) return false;
            II_ResultSet::ChildOffsets &co = rs->child_off[j];
            co.bytes = ch->d_mbytes;
            co.off_pos = ch->d_moff_pos;
            co.off_len = ch->d_moff_len;
        }
        a.bytes[j] = rs->child_off[j].bytes;
        a.off_pos[j] = rs->child_off[j].off_pos;
        a.off_len[j] = rs->child_off[j].off_len;
        a.tag[j] = j < rs->child_tag.size() ? rs->child_tag[j] : 4;
    }
    const uint32_t chunks = (uint32_t)((m + 255) / 256);
    uint32_t *ub = dalloc<uint32_t>(m ? m : 1), *csum = dalloc<uint32_t>(chunks ? chunks : 1), *coff = dalloc<uint32_t>(chunks ? chunks : 1);
    uint32_t *tot32 = dalloc<uint32_t>(4);
    unsigned long long *tot64 = dalloc<unsigned long long>(1);
    dfree(ns->d_moff_pos); // a previous attempt that failed half-way
    dfree(ns->d_moff_len);
    dfree(ns->d_mbytes);
    ns->d_mbytes = nullptr;
    ns->d_moff_pos = dalloc<uint32_t>(m ? m : 1);
    ns->d_moff_len = dalloc<uint32_t>(m ? m : 1);
    bool ok = ub && csum && coff && tot32 && tot64 && ns->d_moff_pos && ns->d_moff_len;
    unsigned long long total = 0;
    ok = ok && ii_launch_merge_offsets_bounds(a, nullptr, (uint32_t)m, ub, csum, coff, tot32, tot64, c.stream) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(&total, tot64, 8, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    ok = ok && total < 0xFFFFFFFFull;
    if (ok) {
        ns->d_mbytes = dalloc<uint8_t>((size_t)total + 16);
        ok = ns->d_mbytes != nullptr;
    }
    ok = ok && ii_launch_merge_offsets_write(a, nullptr, (uint32_t)m, ub, coff, ns->d_mbytes, ns->d_moff_pos, ns->d_moff_len, c.stream) == cudaSuccess;
    c.stats.kernel_launches += 3;
    dfree(ub);
    dfree(csum);
    dfree(coff);
    dfree(tot32);
    dfree(tot64);
    ns->merged = ok;
    return ok;
}

// the offsets tables of the nested children of `rs` (their merged streams), for the kernels that walk term positions
bool ensure_child_offsets(Ctx &c, II_ResultSet *rs) {
    for (uint32_t j = 0; j < rs->n_children && j < rs->nested.size(); j++) {
        if (!rs->nested[j]) continue;
        NestedSet *ch = rs->nested[j].get();
        if (!ensure_merged(c, ch)) return false;
        II_ResultSet::ChildOffsets &co = rs->child_off[j];
        co.bytes = ch->d_mbytes;
        co.off_pos = ch->d_moff_pos;
        co.off_len = ch->d_moff_len;
    }
    return true;
}

// GetSlop per hit, once per result set and only when a legacy scorer asks for it.  d_len / cap_len as for the scorer launch.
bool ensure_slop(Ctx &c, II_ResultSet *rs, const uint32_t *d_len, uint32_t cap_len) {
    if (!rs->d_hit_pos || rs->d_slop) return true;
    if (rs->n_children > (uint32_t)kIIMaxLists) return true;
    if (!ensure_child_offsets(c, rs)) return false;
    rs->d_slop = dalloc<uint32_t>(rs->cap);
    if (!rs->d_slop) return false;
    SlopArgs sa{};
    sa.n = rs->n_children;
    sa.is_union = rs->is_union ? 1 : 0;
    sa.order = rs->d_order;
    sa.pos = rs->d_hit_pos;
    sa.fstride = rs->cap;
    for (uint32_t j = 0; j < rs->n_children; j++) {
        sa.bytes[j] = rs->child_off[j].bytes;
        sa.off_pos[j] = rs->child_off[j].off_pos;
        sa.off_len[j] = rs->child_off[j].off_len;
    }
    c.stats.kernel_launches += 1;
    return ii_launch_min_offset_delta(sa, rs->d_docs, d_len, cap_len, rs->d_slop, c.stream) == cudaSuccess;
}

ScoreArgs make_score_args(II_ResultSet *rs, II_Scorer scorer, const II_TermParams *terms, double agg_weight,
                          const II_IndexStats *stats, const II_DocTable *docs, double min_score, uint64_t tanh_factor) {
    ScoreArgs sa{};
    sa.scorer = (int)scorer;
    sa.is_union = rs->is_union;
    sa.n_children = rs->n_children;
    if (rs->n_children <= (uint32_t)kIIMaxLists) {
        for (uint32_t i = 0; i < rs->n_children; i++) {
            const II_TermParams &t = terms[rs->child_order[i]];
            sa.weight[i] = t.weight;
            sa.idf[i] = t.idf;
            sa.bm25_idf[i] = t.bm25_idf;
        }
    } else { // a wide union: the tables do not fit the kernel arguments (pageable source: staged before the copy call returns)
        const uint32_t n = rs->n_children;
        std::vector<double> ext(3 * (size_t)n);
        for (uint32_t i = 0; i < n; i++) {
            const II_TermParams &t = terms[rs->child_order[i]];
            ext[i] = t.weight;
            ext[n + i] = t.idf;
            ext[2 * (size_t)n + i] = t.bm25_idf;
        }
        if (!rs->d_ext) rs->d_ext = dalloc<double>(ext.size());
        if (rs->d_ext) cudaMemcpyAsync(rs->d_ext, ext.data(), ext.size() * 8, cudaMemcpyHostToDevice, ctx().stream);
        sa.ext = rs->d_ext;
        sa.n_children = rs->d_ext ? n : 0; // no table, no children: the launch scores nothing rather than reading past the inline arrays
    }
    sa.agg_weight = agg_weight;
    sa.avg_doc_len = stats ? stats->avgDocLen : 0.0;
    sa.min_score = min_score;
    sa.tanh_factor = tanh_factor ? tanh_factor : 1;
    sa.doc_len = docs ? docs->d_len : nullptr;
    sa.doc_score = docs ? docs->d_score : nullptr;
    sa.max_freq = docs ? docs->d_maxf : nullptr;
    sa.slop = rs->d_slop; // NULL: no term positions on the device, the kernel uses `children - 1`
    sa.order = rs->d_order;
    for (uint32_t i = 0; i < rs->n_children && i < rs->nested.size() && i < (uint32_t)kIIMaxLists; i++)
        if (rs->nested[i]) sa.sub[i] = rs->nested[i]->d_sub;
    sa.pos = rs->d_hit_pos;
    sa.pstride = rs->cap;
    return sa;
}

// The recursive value of every hit of every nested child of `rs` for `scorer` (ScoreArgs::sub), innermost first.
bool prepare_nested_scores(Ctx &c, II_ResultSet *rs, II_Scorer scorer, const II_IndexStats *stats, const II_DocTable *docs) {
    if (scorer == II_SCORER_DOCSCORE || scorer == II_SCORER_HAMMING) return true;
    for (uint32_t j = 0; j < rs->n_children && j < rs->nested.size(); j++) {
        if (!rs->nested[j]) continue;
        NestedSet *ns = rs->nested[j].get();
        II_ResultSet *in = ns->rs.get();
        if (!in->has_freqs) return false;
        if (!prepare_nested_scores(c, in, scorer, stats, docs)) return false;
        if (!ns->d_sub) ns->d_sub = dalloc<double>(in->len ? in->len : 1);
        if (!ns->d_sub) return false;
        ScoreArgs sa = make_score_args(in, scorer, ns->terms.data(), ns->weight, stats, docs, 0.0, 4);
        sa.sub_only = 1;
        sa.slop = nullptr;
        if (ii_launch_score(sa, in->d_docs, in->d_freqs, in->cap, nullptr, (uint32_t)in->len, ns->d_sub, c.stream) != cudaSuccess) return false;
        c.stats.kernel_launches += 1;
    }
    return true;
}

// Everything about an OR of n lists that the host knows before any kernel runs: the set's shape (children, tags, num_estimated,
// cap), the largest last docId, whether children are nested, whether the hits keep their term positions, and the reference's
// aggregate child order.  Shared by II_Union and II_UnionBatchDevice, so that both build the same sets.
struct UnionPlan {
    uint32_t max_id = 0;
    size_t total_in = 0;
    bool any_nested = false, keep_pos = false, flat_order = false;
    UnionOrder uo{};
};
UnionPlan union_plan(II_PostingList *const *lists, size_t n, int quick_exit, II_ResultSet *rs) {
    UnionPlan p;
    rs->is_union = true;
    rs->has_freqs = !quick_exit;
    init_children(rs, n, 4);
    rs->estimated = 0;
    rs->lo_id = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) {
        if (lists[i]->n) {
            p.max_id = std::max(p.max_id, lists[i]->last_id);
            rs->lo_id = std::min(rs->lo_id, lists[i]->first_id);
        }
        p.total_in += lists[i]->n;
        rs->estimated += lists[i]->estimated; // union_flat.rs:102
        rs->child_tag[i] = lists[i]->result_tag;
        if (lists[i]->nested) {
            rs->nested[i] = lists[i]->nested;
            p.any_nested = true;
        }
    }
    rs->hi_id = p.max_id; // every hit is in a non-empty child (no child at all: lo_id > hi_id)
    rs->cap = std::min<size_t>(p.total_in, (size_t)p.max_id + 1);
    // the reference's aggregate child order (UnionFlat, full mode, read front to back): children live in an "active" array,
    // an exhausted child is swap-removed by the pass that follows the document it ended on (advance_and_find_min,
    // union_flat.rs:218-258; empty children by initialize_children :263-296), positions visited in ascending order and a
    // swapped-in child examined at once.  (Above min_union_iter_heap = 20 children the reference uses UnionHeap, whose
    // aggregate order follows its heap array: same docIds and children, sums may differ in the last bit.)
    p.flat_order = rs->has_freqs && n <= (size_t)kIIUnionFlatMax; // more children: UnionHeap, whose order follows its heap array
    if (p.flat_order && p.total_in) {
        UnionOrder &uo = p.uo;
        std::vector<uint32_t> active(n);
        for (size_t i = 0; i < n; i++) active[i] = (uint32_t)i;
        size_t num_active = n;
        auto sweep = [&](auto &&exhausted) {
            for (size_t i = 0; i < num_active;) {
                if (exhausted(active[i])) {
                    num_active--;
                    if (i < num_active) std::swap(active[i], active[num_active]);
                    continue;
                }
                i++;
            }
        };
        sweep([&](uint32_t ch) { return lists[ch]->n == 0; });
        while (num_active) {
            uint32_t bound = 0xFFFFFFFFu;
            for (size_t i = 0; i < num_active; i++) bound = std::min(bound, lists[active[i]]->last_id);
            const uint32_t e = uo.n_epochs++;
            uo.bound[e] = bound;
            uo.n_active[e] = (uint8_t)num_active;
            for (size_t i = 0; i < num_active; i++) uo.perm[e][i] = (uint8_t)active[i];
            sweep([&](uint32_t ch) { return lists[ch]->last_id == bound; });
        }
    }
    for (size_t i = 0; i < n && n > 1 && n <= (size_t)kIIMaxLists && rs->has_freqs; i++) p.keep_pos |= lists[i]->d_off_len != nullptr;
    p.keep_pos |= p.any_nested;
    if (p.keep_pos)
        for (size_t j = 0; j < n; j++) {
            const II_PostingList *L = lists[j];
            II_ResultSet::ChildOffsets &co = rs->child_off[j];
            if (!L->d_off_len) continue;
            co.bytes = L->d_bytes;
            co.off_pos = L->d_off_pos;
            co.off_len = L->d_off_len;
            co.keep_tables = L->owner;
            co.keep_bytes = L->bytes_owner;
        }
    return p;
}

bool union_enqueue(Ctx &c, II_PostingList *const *lists, size_t n, int quick_exit, II_ResultSet *rs, bool *trivially_empty) {
    const UnionPlan plan = union_plan(lists, n, quick_exit, rs);
    const bool any_nested = plan.any_nested, flat_order = plan.flat_order, keep_pos = plan.keep_pos;
    const UnionOrder &uo = plan.uo;
    if (any_nested && (n > (size_t)kIIMaxLists || quick_exit)) return false; // nested children need the per-child position rows
    *trivially_empty = plan.total_in == 0;
    if (*trivially_empty) return true;
    const uint32_t nwords = plan.max_id / 32 + 1, nblk = (nwords + 31) / 32;
    rs->d_docs = dalloc<uint32_t>(rs->cap);
    rs->d_freqs = dalloc<uint32_t>(rs->has_freqs ? rs->cap * n : 1);
    rs->d_scores = dalloc<double>(rs->cap);
    rs->d_len = dalloc<uint32_t>(4);
    uint32_t *bitmap = dalloc<uint32_t>(nwords), *blocksum = dalloc<uint32_t>(nblk), *blockoff = dalloc<uint32_t>(nblk);
    uint32_t *wordoff = dalloc<uint32_t>(nwords);
    if (flat_order) rs->d_order = dalloc<UnionOrder>(1);
    if (keep_pos) rs->d_hit_pos = dalloc<uint32_t>(rs->cap * n);
    bool ok = rs->d_docs && rs->d_freqs && rs->d_scores && rs->d_len && bitmap && blocksum && blockoff && wordoff &&
              (!flat_order || rs->d_order) && (!keep_pos || rs->d_hit_pos);
    if (ok) {
        std::vector<const uint32_t *> ids(n), freqs(n);
        std::vector<uint32_t> lens(n);
        for (size_t i = 0; i < n; i++) {
            ids[i] = lists[i]->d_ids;
            freqs[i] = lists[i]->d_freqs;
            lens[i] = (uint32_t)lists[i]->n;
        }
        cudaEventRecord(c.e0, c.stream);
        if (rs->has_freqs) ok = cudaMemsetAsync(rs->d_freqs, 0, rs->cap * n * 4, c.stream) == cudaSuccess;
        if (rs->d_order) { // pageable source: the copy is staged before the call returns
            ok = ok && cudaMemcpyAsync(rs->d_order, &uo, sizeof(uo), cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
            rs->h_order.reset(new UnionOrder(uo));
        }
        if (keep_pos) ok = ok && cudaMemsetAsync(rs->d_hit_pos, 0xFF, rs->cap * n * 4, c.stream) == cudaSuccess;
        ok = ok && ii_launch_union(ids.data(), freqs.data(), lens.data(), (uint32_t)n, nwords, bitmap, blocksum, blockoff, wordoff,
                                   rs->d_len, rs->d_docs, rs->d_freqs, rs->cap, rs->has_freqs, rs->d_hit_pos, c.stream) == cudaSuccess;
        cudaEventRecord(c.e1, c.stream);
        c.stats.kernel_launches += 3 + 2 * n;
    }
    dfree(bitmap);
    dfree(blocksum);
    dfree(blockoff);
    dfree(wordoff);
    return ok;
}

// after the stream has been synchronised
void finish_len(Ctx &c, II_ResultSet *rs) {
    rs->len = *c.h_total;
    float ms = 0;
    if (cudaEventElapsedTime(&ms, c.e0, c.e1) == cudaSuccess) c.stats.intersect_device_us = ms * 1000.0;
}

// One set built synchronously on the calling thread's context: `enqueue(c, rs, &trivially_empty)` (intersect_enqueue or
// union_enqueue) queues its kernels, then the count is read back.  NULL where the enqueue or the read-back failed.
extern "C++" template <class Enqueue> II_ResultSet *build_sync(Enqueue &&enqueue) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return nullptr;
    std::unique_ptr<II_ResultSet> rs(new II_ResultSet());
    bool empty = false;
    bool ok = enqueue(c, rs.get(), &empty);
    if (ok && !empty) {
        ok = cudaMemcpyAsync(c.h_total, rs->d_len, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        if (ok) finish_len(c, rs.get());
    }
    return ok ? rs.release() : nullptr;
}

// merge the per-warp top-N lists the device selected (<= lists*k survivors)
size_t merge_topn_lists(const uint64_t *keys, const uint32_t *ids, size_t total, size_t k, uint64_t *doc_ids, double *scores) {
    std::vector<uint32_t> idx;
    for (uint32_t i = 0; i < total; i++)
        if (ids[i] != 0xFFFFFFFFu) idx.push_back(i);
    const size_t kk = std::min<size_t>(k, idx.size());
    std::partial_sort(idx.begin(), idx.begin() + kk, idx.end(), [&](uint32_t a, uint32_t b) {
        return keys[a] < keys[b] || (keys[a] == keys[b] && ids[a] < ids[b]);
    });
    for (size_t i = 0; i < kk; i++) {
        doc_ids[i] = ids[idx[i]];
        uint64_t u = ~keys[idx[i]];
        u = (u >> 63) ? (u & 0x7FFFFFFFFFFFFFFFull) : ~u;
        memcpy(&scores[i], &u, 8);
    }
    return kk;
}

// One fused search in flight on a context: everything enqueued, nothing waited for.
struct PendingSearch {
    bool active = false;
    std::unique_ptr<II_ResultSet> rs;
    uint64_t *h_keys = nullptr;
    uint32_t *h_ids = nullptr;
    size_t total = 0;
    uint32_t k = 0;
};

// AND/OR -> score -> per-warp top-N lists -> D2H, all on c.stream; false (and nothing pending) if the answer is
// trivially empty or a launch failed
bool search_enqueue(Ctx &c, II_PostingList *const *lists, size_t n, int is_union, II_Scorer scorer, const II_TermParams *terms,
                    double agg_weight, const II_IndexStats *stats, const II_DocTable *docs, size_t top_n, PendingSearch &p) {
    p.active = false;
    p.rs.reset(new II_ResultSet());
    II_ResultSet &rs = *p.rs;
    bool empty = false;
    bool ok = is_union ? union_enqueue(c, lists, n, 0, &rs, &empty) : intersect_enqueue(c, lists, n, &rs, &empty);
    if (!ok || empty) {
        p.rs.reset();
        return false;
    }
    const uint32_t k = (uint32_t)top_n;
    if (scorer == II_SCORER_BM25 || scorer == II_SCORER_TFIDF || scorer == II_SCORER_TFIDF_DOCNORM)
        ok = ensure_slop(c, &rs, rs.d_len, (uint32_t)rs.cap);
    ok = ok && prepare_nested_scores(c, &rs, scorer, stats, docs);
    const ScoreArgs sa = make_score_args(&rs, scorer, terms, agg_weight, stats, docs, 0.0, 4);
    ok = ok && ii_launch_score(sa, rs.d_docs, rs.d_freqs, rs.cap, rs.d_len, (uint32_t)rs.cap, rs.d_scores, c.stream) == cudaSuccess;
    const uint32_t nl = ii_topn_lists((uint32_t)rs.cap);
    const size_t total = (size_t)nl * k;
    uint64_t *d_keys = dalloc<uint64_t>(total);
    uint32_t *d_ids = dalloc<uint32_t>(total);
    uint8_t *stg = c.stage(total * 12);
    ok = ok && d_keys && d_ids && stg;
    p.h_keys = reinterpret_cast<uint64_t *>(stg);
    p.h_ids = reinterpret_cast<uint32_t *>(p.h_keys + total);
    ok = ok && ii_launch_topn(rs.d_docs, rs.d_scores, rs.d_len, (uint32_t)rs.cap, k, d_keys, d_ids, c.stream) == cudaSuccess;
    cudaEventRecord(c.e2, c.stream);
    ok = ok && cudaMemcpyAsync(p.h_keys, d_keys, total * 8, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(p.h_ids, d_ids, total * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(c.h_total, rs.d_len, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    dfree(d_keys);
    dfree(d_ids);
    c.stats.kernel_launches += 2;
    if (!ok) {
        cudaStreamSynchronize(c.stream);
        p.rs.reset();
        return false;
    }
    p.total = total;
    p.k = k;
    p.active = true;
    return true;
}

// wait for the context's stream and merge the per-warp lists on the host; must run with `c` current
size_t search_finish(Ctx &c, PendingSearch &p, uint64_t *doc_ids, double *scores, size_t *total_hits) {
    p.active = false;
    if (cudaStreamSynchronize(c.stream) != cudaSuccess) {
        p.rs.reset();
        return 0;
    }
    finish_len(c, p.rs.get());
    float ms = 0;
    if (cudaEventElapsedTime(&ms, c.e1, c.e2) == cudaSuccess) c.stats.score_device_us = ms * 1000.0;
    const size_t len = p.rs->len;
    if (total_hits) *total_hits = len;
    const size_t got = merge_topn_lists(p.h_keys, p.h_ids, p.total, std::min<size_t>(p.k, len), doc_ids, scores);
    p.rs.reset(); // stream-ordered frees on c.stream
    return got;
}

} // namespace

II_ResultSet *II_Intersect(II_PostingList *const *lists, size_t n) { return II_IntersectEx(lists, nullptr, n); }

// AND with NOT / OPTIONAL children: modes[i] 0 = required, 1 = NOT (docIds of lists[i] are excluded), 2 = OPTIONAL (never
// rejects; its freq is kept where present).  The excluded / absent children yield virtual results (freq 0, score 0).
II_ResultSet *II_IntersectEx(II_PostingList *const *lists, const int *modes, size_t n) {
    if (n == 0 || n > (size_t)kIIMaxLists) return nullptr;
    return build_sync([&](Ctx &c, II_ResultSet *rs, bool *empty) { return intersect_enqueue(c, lists, n, rs, empty, modes); });
}

// AND with the reference's proximity constraints (intersection.rs:201-242 -> index_result proximity.rs): max_slop < 0 = no
// limit; in_order = the terms must appear in the order of `lists` (which is then also the aggregate child order).  Every
// required / optional list must carry term positions (II_PostingList_FromBlocksBatchOffsets, Full codec).
II_ResultSet *II_IntersectPhrase(II_PostingList *const *lists, const int *modes, size_t n, int32_t max_slop, int in_order) {
    if (n == 0 || n > (size_t)kPhraseMaxLists) return nullptr;
    for (size_t i = 0; i < n; i++)
        if ((!modes || modes[i] != 1) && !lists[i]->d_off_len) return nullptr;
    const PhraseSpec ph{max_slop < 0 ? 0xFFFFFFFFu : (uint32_t)max_slop, in_order != 0};
    const bool constrained = max_slop >= 0 || in_order;
    return build_sync(
        [&](Ctx &c, II_ResultSet *rs, bool *empty) { return intersect_enqueue(c, lists, n, rs, empty, modes, constrained ? &ph : nullptr); });
}

// nq independent ANDs in one call (the filters of a batch of hybrid queries): every intersection is enqueued on its own stream
// before anything is waited for; out[i] = NULL where it could not be built (an empty child yields an empty result set).
size_t II_IntersectBatch(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, II_ResultSet **out) {
    constexpr size_t kSlots = 16;
    struct Pool {
        std::mutex mu;
        Ctx slot[kSlots];
    };
    static Pool pool;
    std::lock_guard<std::mutex> g(pool.mu);
    size_t built = 0;
    for (size_t q0 = 0; q0 < nq; q0 += kSlots) {
        const size_t q1 = std::min(nq, q0 + kSlots);
        bool pending[kSlots] = {false};
        for (size_t qi = q0; qi < q1; qi++) {
            out[qi] = nullptr;
            const size_t sl = qi - q0, n = n_lists[qi];
            if (n == 0 || n > (size_t)kIIMaxLists) continue;
            CtxScope scope(&pool.slot[sl]);
            Ctx &c = pool.slot[sl];
            if (!c.init()) continue;
            auto *rs = new II_ResultSet();
            bool empty = false;
            bool ok = intersect_enqueue(c, lists[qi], n, rs, &empty);
            if (ok && !empty) {
                ok = cudaMemcpyAsync(c.h_total, rs->d_len, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
                pending[sl] = ok;
            }
            if (!ok) {
                cudaStreamSynchronize(c.stream);
                delete rs;
                continue;
            }
            out[qi] = rs;
        }
        for (size_t qi = q0; qi < q1; qi++) {
            const size_t sl = qi - q0;
            if (!out[qi]) continue;
            CtxScope scope(&pool.slot[sl]);
            Ctx &c = pool.slot[sl];
            if (pending[sl]) {
                if (cudaStreamSynchronize(c.stream) != cudaSuccess) {
                    delete out[qi];
                    out[qi] = nullptr;
                    continue;
                }
                finish_len(c, out[qi]);
            }
            built++;
        }
    }
    return built;
}

// The same ANDs with no host wait: round-robin over a pool of streams of their own, each set's count left in its d_len, and
// `stream` made to wait for every stream used.  A set stays `pending` until an accessor needs its length on the host (settle).
size_t II_IntersectBatchDevice(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, void *stream, II_ResultSet **out) {
    constexpr size_t kSlots = 16;
    struct Pool {
        std::mutex mu;
        Ctx slot[kSlots];
        cudaEvent_t done[kSlots] = {};
    };
    static Pool pool;
    std::lock_guard<std::mutex> g(pool.mu);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    bool used[kSlots] = {false};
    size_t built = 0;
    for (size_t qi = 0; qi < nq; qi++) {
        out[qi] = nullptr;
        const size_t sl = qi % kSlots, n = n_lists[qi];
        if (n == 0 || n > (size_t)kIIMaxLists) continue;
        CtxScope scope(&pool.slot[sl]); // the set's memory is allocated and, on failure, freed in this stream's order
        Ctx &c = pool.slot[sl];
        if (!c.init()) continue;
        std::unique_ptr<II_ResultSet> rs(new II_ResultSet());
        bool empty = false;
        if (!intersect_enqueue(c, lists[qi], n, rs.get(), &empty) || empty) continue;
        if (cudaEventCreateWithFlags(&rs->ready, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(rs->ready, c.stream) != cudaSuccess)
            continue;
        rs->pending = true;
        used[sl] = true;
        out[qi] = rs.release();
        built++;
    }
    for (size_t sl = 0; sl < kSlots; sl++) {
        if (!used[sl]) continue;
        if (!pool.done[sl] && cudaEventCreateWithFlags(&pool.done[sl], cudaEventDisableTiming) != cudaSuccess) continue;
        // the wait takes the event's state now: re-recording it for the next batch does not move this wait
        if (cudaEventRecord(pool.done[sl], pool.slot[sl].stream) == cudaSuccess) cudaStreamWaitEvent(st, pool.done[sl], 0);
    }
    return built;
}

namespace {
// a pending set (II_IntersectBatchDevice): wait for its AND, then its length is on the host as for every other set
void settle(const II_ResultSet *crs) {
    if (!crs || !crs->pending) return;
    static std::mutex mu;
    static cudaStream_t s = nullptr; // of its own: the copy queues behind nothing but the set's AND
    std::lock_guard<std::mutex> g(mu);
    auto *rs = const_cast<II_ResultSet *>(crs);
    if (!rs->pending) return;
    if (!s && cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return;
    uint32_t len[2 + kIIMaxLists] = {};
    const size_t words = (rs->estimated_on_device ? 2 : 1) + rs->order_weight.size(); // a deferred child order: estimated on device
    if (cudaStreamWaitEvent(s, rs->ready, 0) != cudaSuccess ||
        cudaMemcpyAsync(len, rs->d_len, words * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)
        return;
    rs->len = len[0];
    if (rs->estimated_on_device) rs->estimated = len[1];
    if (!rs->order_weight.empty()) { // Intersection::new's order over the children's estimates, now on the host
        const std::vector<double> &w = rs->order_weight;
        and_order(rs, w.size(), [&](size_t i) { return AndKey{w[i] >= 0, (double)len[2 + i], w[i]}; });
        rs->order_weight.clear();
    }
    rs->pending = false;
}
} // namespace

const uint32_t *II_ResultSet_DeviceLen(const II_ResultSet *rs) { return rs->d_len; }
size_t II_ResultSet_Capacity(const II_ResultSet *rs) { return rs->cap; }

void II_ResultSet_FreeAfter(II_ResultSet *rs, void *stream) {
    if (!rs) return;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    cudaEvent_t ev = nullptr;
    if (c.init() && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess) {
        // the frees of the destructor run in c.stream order: after everything enqueued on `stream` so far (and the AND itself)
        if (cudaEventRecord(ev, st) == cudaSuccess) cudaStreamWaitEvent(c.stream, ev, 0);
        cudaEventDestroy(ev);
    } else {
        cudaStreamSynchronize(st);
    }
    delete rs;
}

II_ResultSet *II_Union(II_PostingList *const *lists, size_t n, int quick_exit) {
    if (n == 0 || n > (size_t)kIIMaxUnionLists) return nullptr;
    return build_sync([&](Ctx &c, II_ResultSet *rs, bool *empty) { return union_enqueue(c, lists, n, quick_exit, rs, empty); });
}

namespace {
// A batch call that reads child sets: c.stream waits for each one's own kernels once (a settled or host-built set: at once).
// inputs is sorted and made unique.
bool wait_for_inputs(Ctx &c, std::vector<II_ResultSet *> &inputs) {
    std::sort(inputs.begin(), inputs.end());
    inputs.erase(std::unique(inputs.begin(), inputs.end()), inputs.end());
    bool ok = true;
    for (II_ResultSet *s : inputs)
        if (s->ready) ok = ok && cudaStreamWaitEvent(c.stream, s->ready, 0) == cudaSuccess;
    return ok;
}
// every input keeps the call's completion event (recorded now on c.stream): its memory is not handed out again while the call's
// kernels may still read it, whichever thread frees it
bool borrow_inputs(Ctx &c, const std::vector<II_ResultSet *> &inputs) {
    auto done = std::make_shared<SharedEvent>();
    if (cudaEventCreateWithFlags(&done->ev, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(done->ev, c.stream) != cudaSuccess) {
        cudaStreamSynchronize(c.stream);
        return false;
    }
    std::lock_guard<std::mutex> rg(readers_mu());
    for (II_ResultSet *s : inputs) {
        auto &r = s->readers;
        r.erase(std::remove_if(r.begin(), r.end(), [](const std::shared_ptr<SharedEvent> &e) { return cudaEventQuery(e->ev) == cudaSuccess; }),
                r.end());
        r.push_back(done);
    }
    cudaGetLastError(); // cudaErrorNotReady of a reader still running is no failure
    return true;
}

// The part of a batch plan that publish_pending hands out: the set built for query q
struct PendingPlan {
    size_t q;
    std::unique_ptr<II_ResultSet> rs;
};
// The end of a batch call that hands out pending sets, once their memory, the device buffer `d_buf` and the pinned `slot` are
// allocated and the tables filled in the slot (ok: all of that succeeded).  The first tab_bytes of the slot go up to d_buf in one
// copy, `launch` runs once every input set's own kernels are done, and the inputs are borrowed: each keeps the call's completion
// event, which its destructor waits for.  d_buf is freed in stream order, an event per set marks it pending, `stream` waits for
// the last one and out[q] / *built receive the sets.  On failure nothing is handed out and the result is -1.
extern "C++" template <class Plan, class Launch>
int publish_pending(Ctx &c, bool ok, Ctx::UploadSlot *slot, uint8_t *d_buf, size_t tab_bytes, std::vector<II_ResultSet *> &inputs,
                    Launch &&launch, std::vector<Plan> &plans, void *stream, II_ResultSet **out, size_t *built) {
    if (ok) {
        ok = wait_for_inputs(c, inputs);
        ok = ok && cudaMemcpyAsync(d_buf, slot->h, tab_bytes, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        ok = ok && cudaEventRecord(slot->ev, c.stream) == cudaSuccess;
        ok = ok && launch();
        if (!inputs.empty()) ok = borrow_inputs(c, inputs) && ok;
    }
    dfree(d_buf);
    for (Plan &p : plans) {
        II_ResultSet *rs = p.rs.get();
        ok = ok && cudaEventCreateWithFlags(&rs->ready, cudaEventDisableTiming) == cudaSuccess && cudaEventRecord(rs->ready, c.stream) == cudaSuccess;
        rs->pending = true;
    }
    if (!ok) { // a failed allocation or launch: nothing is handed out (the frees run in c.stream order behind whatever was enqueued)
        cudaGetLastError();
        return -1;
    }
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    // every set's event completes at the same point of c.stream: waiting for the last one waits for the whole batch
    if (cudaStreamWaitEvent(st, plans.back().rs->ready, 0) != cudaSuccess) {
        cudaStreamSynchronize(c.stream);
        return -1;
    }
    for (Plan &p : plans) out[p.q] = p.rs.release();
    if (built) *built = plans.size();
    return 0;
}

// The shape II_Union(quick) gives a filter-mode OR of n children: docIds only, identity child order, every child tagged `tag`
void filter_union_shape(II_ResultSet *rs, size_t n, uint8_t tag) {
    rs->is_union = true;
    rs->has_freqs = false;
    init_children(rs, n, tag);
}

// One child of a batch OR as the kernels see it: a posting list, a numeric leaf or a set.  len: the exact length of a list or a
// leaf, a set's capacity (its count is read on the device, d_len); [lo, hi]: host-known bounds on its docIds.
struct OrChild {
    const uint32_t *ids = nullptr, *freqs = nullptr, *d_len = nullptr, *d_est = nullptr;
    const double *values = nullptr;
    size_t len = 0;
    uint32_t lo = 0, hi = 0;
};

// A batch of ORs with no host wait, over one of three kinds of children: posting lists (II_UnionBatchDevice), numeric leaves
// filtered by a range (II_NumericFilterBatchDevice), or filter children, lists and sets (II_UnionFilterBatchDevice).  Every set's
// memory comes from the pool in c.stream order and ii_launch_union_batch runs the same 4 or 6 launches for any batch; the upload,
// the borrowed child sets and the pending sets are publish_pending's.
int filter_batch_device(size_t nq, II_PostingList *const *const *lists, II_NumericList *const *const *leaves,
                        const II_FilterChild *const *children, const size_t *counts, int quick_exit, const II_NumericRange *ranges,
                        void *stream, II_ResultSet **out, size_t *built) {
    const bool numeric = leaves != nullptr, sets = children != nullptr, full = !numeric && !sets && !quick_exit;
    const void *const *tab = numeric ? (const void *const *)leaves : sets ? (const void *const *)children : (const void *const *)lists;
    if (built) *built = 0;
    if (nq && (!out || !counts || !tab)) return -1;
    for (size_t q = 0; q < nq; q++) out[q] = nullptr;
    for (size_t q = 0; q < nq; q++) { // refused before anything is enqueued
        if (counts[q] > (size_t)kIIMaxUnionLists || (counts[q] && !tab[q])) return -1;
        if (numeric && !ranges) return -1;
        for (size_t i = 0; i < counts[q]; i++) {
            if (sets) {
                const II_FilterChild &ch = children[q][i];
                if (ch.mode != 0 || (ch.list && ch.set)) return -1;
            } else if (numeric ? !leaves[q][i] : (!lists[q][i] || lists[q][i]->nested)) {
                return -1;
            }
        }
    }
    for (size_t q = 0; sets && q < nq; q++) // the children are read only once every argument passed the checks above
        for (size_t i = 0; i < counts[q]; i++)
            if (children[q][i].list && children[q][i].list->nested) return -1;
    const auto child = [&](size_t q, size_t i) {
        OrChild e;
        const II_PostingList *pl = sets ? children[q][i].list : numeric ? nullptr : lists[q][i];
        const II_ResultSet *s = sets ? children[q][i].set : nullptr;
        if (numeric) {
            const II_NumericList *nl = leaves[q][i];
            e.ids = nl->d_ids;
            e.values = nl->d_values;
            e.len = nl->n;
            e.lo = nl->first_id;
            e.hi = nl->last_id;
        } else if (pl) {
            e.ids = pl->d_ids;
            e.freqs = full ? pl->d_freqs : nullptr;
            e.len = pl->n;
            e.lo = pl->first_id;
            e.hi = pl->last_id;
        } else if (s && s->cap) { // a set built empty may have no device count
            e.ids = s->d_docs;
            e.d_len = s->d_len;
            e.d_est = s->pending && s->estimated_on_device ? s->d_len + 1 : nullptr;
            e.len = s->cap;
            e.lo = s->lo_id;
            e.hi = s->hi_id;
        }
        return e;
    };
    struct Plan : PendingPlan {
        uint32_t lo_word, nwords, nblk;
        uint64_t blk0;
        bool keep_pos;
        UnionOrder uo;
        uint64_t est_host; // sets: the sum of the estimates known on the host, saturated
        uint32_t n_est_dev;
    };
    std::vector<Plan> plans;
    std::vector<II_ResultSet *> inputs; // every child set, once
    uint64_t total_blocks = 0, total_chunks = 0, clear_elems = 0;
    size_t nlists = 0, n_orders = 0, n_est_dev = 0;
    for (size_t q = 0; q < nq; q++) {
        const size_t n = counts[q];
        if (!n) continue;
        Plan p{{q, std::unique_ptr<II_ResultSet>(new II_ResultSet())}, 0, 0, 0, 0, false, UnionOrder{}, 0, 0};
        II_ResultSet *rs = p.rs.get();
        uint32_t lo = 0xFFFFFFFFu, hi = 0; // the window: over the children that can hold a docId
        size_t total_in = 0;
        for (size_t i = 0; i < n; i++) {
            const OrChild e = child(q, i);
            if (!e.len) continue;
            if (e.len > 0xFFFFFFFFu) return -1; // not representable in the 32-bit tables
            if (e.lo <= e.hi) {
                lo = std::min(lo, e.lo);
                hi = std::max(hi, e.hi);
            }
            total_in += e.len;
            total_chunks += (e.len + kUBChunk - 1) / kUBChunk;
            nlists++;
        }
        if (numeric) { // the shape of II_Union(quick) over II_NumericList_Filter of every leaf
            filter_union_shape(rs, n, 16);
            rs->cap = std::min<size_t>(total_in, (size_t)hi + 1);
            rs->estimated_on_device = true;
        } else if (sets) { // the shape union_plan gives a quick union over the lists plus a list view of each set
            filter_union_shape(rs, n, 4);
            size_t est = 0;
            for (size_t i = 0; i < n; i++) {
                const II_FilterChild &ch = children[q][i];
                if (ch.set) inputs.push_back(const_cast<II_ResultSet *>(ch.set)); // borrowed: only its reader events change
                if (ch.list) rs->child_tag[i] = ch.list->result_tag;
                if (ch.set) rs->child_tag[i] = ch.set->is_union ? 1 : 2; // an OR or a numeric set 1, an AND 2 (IntoChild's tags)
                if (child(q, i).d_est) p.n_est_dev++;
                else est += ch.list ? ch.list->estimated : ch.set ? ch.set->estimated : 0; // union_flat.rs:102
            }
            rs->estimated = est;
            rs->estimated_on_device = p.n_est_dev != 0; // the sum waits for the device: settle() reads it from d_len[1]
            p.est_host = std::min<uint64_t>(est, 0xFFFFFFFFu);
            n_est_dev += p.n_est_dev;
            rs->cap = std::min<size_t>(total_in, (size_t)hi + 1);
        } else {
            const UnionPlan up = union_plan(lists[q], n, quick_exit, rs);
            p.keep_pos = up.keep_pos;
            if (up.flat_order) {
                p.uo = up.uo;
                rs->h_order.reset(new UnionOrder(up.uo));
                n_orders++;
            }
        }
        rs->lo_id = lo;
        rs->hi_id = hi;
        if (!total_in) continue; // nothing can match: no set
        if (lo > hi) lo = hi = 0; // no child can hold a docId (an AND whose bounds exclude each other): a one-block window
        p.lo_word = lo / 32;
        p.nwords = hi / 32 - p.lo_word + 1;
        p.nblk = (p.nwords + 31) / 32;
        p.blk0 = total_blocks;
        total_blocks += p.nblk;
        if (full) clear_elems = std::max<uint64_t>(clear_elems, (uint64_t)rs->cap * n);
        plans.push_back(std::move(p));
    }
    if (plans.empty()) return 0;
    if (total_chunks > 0x7FFFFFFFull || plans.size() > 0xFFFFFFFFull) return -1;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return -1;
    // per-set memory, then the batch's tables and bitmap scratch in one buffer (freed by publish_pending in stream order)
    bool ok = true;
    for (Plan &p : plans) {
        II_ResultSet *rs = p.rs.get();
        const size_t n = counts[p.q];
        rs->d_docs = dalloc<uint32_t>(rs->cap);
        rs->d_freqs = dalloc<uint32_t>(full ? rs->cap * n : 1);
        rs->d_scores = dalloc<double>(rs->cap);
        rs->d_len = dalloc<uint32_t>(4);
        if (rs->h_order) rs->d_order = dalloc<UnionOrder>(1);
        if (p.keep_pos) rs->d_hit_pos = dalloc<uint32_t>(rs->cap * n);
        ok = ok && rs->d_docs && rs->d_freqs && rs->d_scores && rs->d_len && (!rs->h_order || rs->d_order) && (!p.keep_pos || rs->d_hit_pos);
    }
    const size_t nb = plans.size();
    const uint64_t total_words = total_blocks * 32;
    struct Layout {
        UBList *lists;
        UBQuery *q;
        UnionOrder *orders;
        const uint32_t **est_dev;
        size_t tab_bytes; // the tables above: what the pinned slot holds and the upload copies
        uint32_t *est, *bitmap, *blocksum, *blockoff, *wordoff;
        size_t bytes;
    };
    const auto layout = [&](void *base, bool tables_only) {
        BatchScratch s(base);
        Layout L{};
        L.lists = s.take<UBList>(nlists);
        L.q = s.take<UBQuery>(nb);
        L.orders = s.take<UnionOrder>(n_orders);
        L.est_dev = s.take<const uint32_t *>(n_est_dev);
        L.tab_bytes = s.bytes();
        if (tables_only) return L;
        // ii_launch_union_batch clears [est, bitmap + total_words) with one memset: the estimate words must come from this
        // buffer, right before the bitmap
        L.est = s.take<uint32_t>(nb);
        L.bitmap = s.take<uint32_t>(total_words);
        L.blocksum = s.take<uint32_t>(total_blocks);
        L.blockoff = s.take<uint32_t>(total_blocks);
        L.wordoff = s.take<uint32_t>(full ? total_words : 0);
        L.bytes = s.bytes();
        return L;
    };
    const Layout size = layout(nullptr, false);
    uint8_t *d_buf = ok ? dalloc<uint8_t>(size.bytes) : nullptr;
    Ctx::UploadSlot *slot = ok ? c.upload_slot(size.tab_bytes) : nullptr;
    ok = ok && d_buf && slot;
    Layout h{}, d{};
    if (ok) {
        h = layout(slot->h, true);
        d = layout(d_buf, false);
        uint32_t li = 0, chunk = 0, oi = 0, ei = 0;
        for (size_t b = 0; b < nb; b++) {
            const Plan &p = plans[b];
            II_ResultSet *rs = p.rs.get();
            const size_t n = counts[p.q];
            UBQuery &Q = h.q[b];
            Q = UBQuery{};
            Q.docs = rs->d_docs;
            Q.freqs = full ? rs->d_freqs : nullptr;
            Q.pos = rs->d_hit_pos;
            Q.len = rs->d_len;
            if (rs->h_order) {
                h.orders[oi] = p.uo;
                Q.order = rs->d_order;
                Q.order_src = d.orders + oi++;
            }
            Q.blk0 = p.blk0;
            Q.nblk = p.nblk;
            Q.lo_word = p.lo_word;
            Q.nwords = p.nwords;
            Q.n_rows = (uint32_t)n;
            Q.cap = rs->cap;
            if (numeric) {
                const II_NumericRange &r = ranges[p.q];
                Q.mn = r.min;
                Q.mx = r.max;
                Q.mni = r.min_inclusive != 0;
                Q.mxi = r.max_inclusive != 0;
            }
            if (sets) {
                Q.sum_est = 1;
                Q.est_host = p.est_host;
                Q.est_dev = d.est_dev + ei;
                Q.n_est_dev = p.n_est_dev;
            }
            for (size_t i = 0; i < n; i++) {
                const OrChild e = child(p.q, i);
                if (e.d_est) h.est_dev[ei++] = e.d_est;
                if (!e.len) continue;
                h.lists[li] = UBList{e.ids, e.freqs, e.values, e.d_len, (uint32_t)e.len, (uint32_t)b, (uint32_t)i, chunk};
                chunk += (uint32_t)((e.len + kUBChunk - 1) / kUBChunk);
                li++;
            }
        }
    }
    const auto launch = [&] {
        uint32_t launches = 0;
        const bool r = ii_launch_union_batch(d.lists, (uint32_t)nlists, (uint32_t)total_chunks, d.q, (uint32_t)nb, total_blocks, clear_elems,
                                             d.est, d.bitmap, d.blocksum, d.blockoff, d.wordoff, &launches, c.stream) == cudaSuccess;
        c.stats.kernel_launches += launches;
        return r;
    };
    return publish_pending(c, ok, slot, d_buf, size.tab_bytes, inputs, launch, plans, stream, out, built);
}
} // namespace

int II_UnionBatchDevice(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, int quick_exit, void *stream,
                        II_ResultSet **out, size_t *built) {
    return filter_batch_device(nq, lists, nullptr, nullptr, n_lists, quick_exit, nullptr, stream, out, built);
}

int II_NumericFilterBatchDevice(size_t nq, II_NumericList *const *const *leaves, const size_t *n_leaves, const II_NumericRange *ranges,
                                void *stream, II_ResultSet **out, size_t *built) {
    return filter_batch_device(nq, nullptr, leaves, nullptr, n_leaves, 1, ranges, stream, out, built);
}

// ORs over lists and (pending) sets in filter mode, with no host wait: the union batch above with each set's count read on the
// device, and the OR's estimate summed there when a child's is still on the device.
int II_UnionFilterBatchDevice(size_t nq, const II_FilterChild *const *children, const size_t *n_children, void *stream,
                              II_ResultSet **out, size_t *built) {
    return filter_batch_device(nq, nullptr, nullptr, children, n_children, 1, nullptr, stream, out, built);
}

// ANDs over lists and (pending) sets in filter mode, with no host wait.  The driver of each query is the required child with the
// smallest host bound; every other child is probed with the AND of intersect_kernel, each set's count read on the device.  Every
// set's memory comes from the pool in c.stream order and ii_launch_filter_and_batch runs the same 3 launches for any batch; the
// upload, the borrowed child sets and the pending sets are publish_pending's.
int II_IntersectFilterBatchDevice(size_t nq, const II_FilterChild *const *children, const size_t *n_children, void *stream,
                                  II_ResultSet **out, size_t *built) {
    if (built) *built = 0;
    if (nq && (!children || !n_children || !out)) return -1;
    for (size_t q = 0; q < nq; q++) out[q] = nullptr;
    for (size_t q = 0; q < nq; q++) { // refused before anything is enqueued
        const size_t n = n_children[q];
        if (n > (size_t)kIIMaxLists || (n && !children[q])) return -1;
        size_t required = 0;
        for (size_t i = 0; i < n; i++) {
            const II_FilterChild &ch = children[q][i];
            if ((ch.mode != 0 && ch.mode != 1) || (ch.list && ch.set)) return -1;
            required += ch.mode == 0;
        }
        if (!required) return -1;
    }
    const auto bound = [](const II_FilterChild &ch) -> size_t { return ch.list ? ch.list->n : ch.set ? ch.set->cap : 0; };
    const auto sat = [](size_t v) { return (uint32_t)std::min<size_t>(v, 0xFFFFFFFFu); };
    struct Plan : PendingPlan {
        std::vector<uint32_t> probe; // kernel order: the driver, then the others by ascending host bound
        uint32_t chunk0, nchunks;
    };
    std::vector<Plan> plans;
    std::vector<II_ResultSet *> inputs; // every child set, once
    uint64_t total_chunks = 0;
    size_t total_children = 0;
    for (size_t q = 0; q < nq; q++) {
        const size_t n = n_children[q];
        const II_FilterChild *cs = children[q];
        size_t drv = n;
        bool empty = false;
        for (size_t i = 0; i < n; i++) {
            if (cs[i].set) inputs.push_back(const_cast<II_ResultSet *>(cs[i].set)); // borrowed: only its reader events change
            if (cs[i].mode != 0) continue;
            empty |= bound(cs[i]) == 0;
            if (drv == n || bound(cs[i]) < bound(cs[drv])) drv = i;
        }
        if (empty) continue; // a required child empty on the host: no set
        Plan p{{q, std::unique_ptr<II_ResultSet>(new II_ResultSet())}, {}, (uint32_t)total_chunks, 0};
        II_ResultSet *rs = p.rs.get();
        rs->is_union = false;
        rs->has_freqs = false;
        rs->cap = bound(cs[drv]);
        // the shape Intersection::new gives the children: a set counts as the list view II_ResultSet_IntoChild makes of it
        init_children(rs, n, 4);
        std::vector<double> weight(n);
        std::vector<size_t> est(n);
        bool deferred = false;
        rs->estimated = (size_t)-1;
        for (size_t i = 0; i < n; i++) {
            const II_FilterChild &ch = cs[i];
            const II_ResultSet *s = ch.set;
            rs->child_tag[i] = ch.mode == 1 ? 8 : ch.list ? ch.list->result_tag : s->is_union ? 1 : 2;
            weight[i] = ch.list ? ch.list->sort_weight : s && !s->is_union ? 1.0 / (double)std::max<uint32_t>(1, s->n_children) : 1.0;
            est[i] = ch.list ? ch.list->estimated : s ? s->estimated : 0;
            if (ch.mode != 0) continue;
            deferred |= s && s->pending && s->estimated_on_device;
            rs->estimated = std::min(rs->estimated, est[i]);
            rs->lo_id = std::max(rs->lo_id, ch.list ? ch.list->first_id : s->lo_id); // every hit is in each required child
            rs->hi_id = std::min(rs->hi_id, ch.list ? ch.list->last_id : s->hi_id);
        }
        if (deferred) { // the order and the estimate wait for settle()
            rs->estimated_on_device = true;
            rs->order_weight.resize(n);
            for (size_t i = 0; i < n; i++) rs->order_weight[i] = cs[i].mode == 0 ? weight[i] : -1.0;
        } else {
            and_order(rs, n, [&](size_t i) { return AndKey{cs[i].mode == 0, (double)est[i], weight[i]}; });
        }
        p.probe.push_back((uint32_t)drv);
        for (size_t i = 0; i < n; i++)
            if (i != drv) p.probe.push_back((uint32_t)i);
        std::stable_sort(p.probe.begin() + 1, p.probe.end(), [&](uint32_t a, uint32_t b) { return bound(cs[a]) < bound(cs[b]); });
        p.nchunks = (uint32_t)((rs->cap + kIIChunk - 1) / kIIChunk);
        total_chunks += p.nchunks;
        total_children += n;
        plans.push_back(std::move(p));
    }
    if (plans.empty()) return 0;
    if (total_chunks > 0x7FFFFFFFull) return -1;
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return -1;
    // per-set memory, then the batch's tables and scratch in one buffer (freed by publish_pending in stream order)
    bool ok = true;
    for (Plan &p : plans) {
        II_ResultSet *rs = p.rs.get();
        rs->d_docs = dalloc<uint32_t>(rs->cap);
        rs->d_scores = dalloc<double>(rs->cap);
        rs->d_len = dalloc<uint32_t>(2 + (size_t)rs->n_children);
        ok = ok && rs->d_docs && rs->d_scores && rs->d_len;
    }
    const size_t nb = plans.size();
    struct Layout {
        IFBQuery *q;
        IFBChild *children;
        size_t tab_bytes; // the tables above: what the pinned slot holds and the upload copies
        uint32_t *surv, *counts, *offsets;
        size_t bytes;
    };
    const auto layout = [&](void *base, bool tables_only) {
        BatchScratch s(base);
        Layout L{};
        L.q = s.take<IFBQuery>(nb);
        L.children = s.take<IFBChild>(total_children);
        L.tab_bytes = s.bytes();
        if (tables_only) return L;
        L.surv = s.take<uint32_t>((size_t)total_chunks * kIIChunk);
        L.counts = s.take<uint32_t>(total_chunks);
        L.offsets = s.take<uint32_t>(total_chunks);
        L.bytes = s.bytes();
        return L;
    };
    const Layout size = layout(nullptr, false);
    uint8_t *d_buf = ok ? dalloc<uint8_t>(size.bytes) : nullptr;
    Ctx::UploadSlot *slot = ok ? c.upload_slot(size.tab_bytes) : nullptr;
    ok = ok && d_buf && slot;
    Layout d{};
    if (ok) {
        const Layout h = layout(slot->h, true);
        d = layout(d_buf, false);
        uint32_t ci = 0;
        for (size_t b = 0; b < nb; b++) {
            const Plan &p = plans[b];
            II_ResultSet *rs = p.rs.get();
            h.q[b] = IFBQuery{rs->d_docs, rs->d_len, ci, rs->n_children, p.chunk0, p.nchunks};
            for (uint32_t slot_i : p.probe) {
                const II_FilterChild &ch = children[p.q][slot_i];
                IFBChild &K = h.children[ci++];
                K = IFBChild{};
                K.slot = slot_i;
                K.mode = (uint32_t)ch.mode;
                if (ch.list) {
                    K.ids = ch.list->d_ids;
                    K.len = (uint32_t)ch.list->n;
                    K.est = sat(ch.list->estimated);
                } else if (ch.set) {
                    const II_ResultSet *s = ch.set;
                    K.ids = s->d_docs;
                    K.d_len = s->cap ? s->d_len : nullptr; // a set built empty may have no device count
                    K.len = (uint32_t)s->cap;
                    K.d_est = K.d_len && s->pending && s->estimated_on_device ? s->d_len + 1 : nullptr;
                    K.est = sat(s->estimated);
                }
            }
        }
    }
    const auto launch = [&] {
        c.stats.kernel_launches += 3;
        return ii_launch_filter_and_batch(d.children, d.q, (uint32_t)nb, (uint32_t)total_chunks, d.surv, d.counts, d.offsets, c.stream) ==
               cudaSuccess;
    };
    return publish_pending(c, ok, slot, d_buf, size.tab_bytes, inputs, launch, plans, stream, out, built);
}

size_t II_ResultSet_Len(const II_ResultSet *rs) {
    settle(rs);
    return rs->len;
}
size_t II_ResultSet_NumChildren(const II_ResultSet *rs) { return rs->n_children; }
void II_ResultSet_ChildOrder(const II_ResultSet *rs, uint32_t *child_order) {
    if (!rs->order_weight.empty()) settle(rs); // the order waits for the children's estimates on the device
    for (uint32_t i = 0; i < rs->n_children; i++) child_order[i] = rs->child_order[i];
}
void II_ResultSet_Free(II_ResultSet *rs) { delete rs; }

// An evaluated AND / OR becomes ONE child of another aggregate (`(a|b) c`): the list view of its hits (docIds, freq = the sum of
// its children's) that II_Intersect* / II_Union take, carrying the set itself so that the scorers recurse into it and the
// proximity checks / GetSlop see its merged term positions.  CONSUMES rs (also on failure).  terms: of rs's children in the order
// they were given to its constructor; weight: the nested node's own.  with_positions: build the merged positions now (a parent
// with slop / in-order needs them up front; GetSlop builds them on demand).
II_PostingList *II_ResultSet_IntoChild(II_ResultSet *rs, const II_TermParams *terms, double weight, int with_positions) {
    if (!rs) return nullptr;
    settle(rs);
    auto ns = std::make_shared<NestedSet>();
    ns->rs.reset(rs);
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init() || !rs->has_freqs || !terms) return nullptr;
    ns->terms.assign(terms, terms + rs->n_children);
    ns->weight = weight;
    const size_t m = rs->len;
    ns->d_fsum = dalloc<uint32_t>(m ? m : 1);
    bool ok = ns->d_fsum != nullptr;
    ok = ok && ii_launch_sum_freq_rows(rs->d_freqs, rs->n_children, rs->cap, nullptr, (uint32_t)m, ns->d_fsum, c.stream) == cudaSuccess;
    c.stats.kernel_launches += 1;
    uint32_t last = 0;
    if (ok && m) ok = cudaMemcpyAsync(&last, rs->d_docs + m - 1, 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    if (ok && with_positions) ok = ensure_merged(c, ns.get());
    if (!ok) return nullptr;
    auto *pl = new II_PostingList();
    pl->d_ids = rs->d_docs;
    pl->d_freqs = ns->d_fsum;
    pl->n = m;
    pl->estimated = rs->estimated;
    pl->last_id = last;
    pl->result_tag = rs->is_union ? 1 : 2;
    pl->sort_weight = rs->is_union ? 1.0 : 1.0 / (double)std::max<uint32_t>(1, rs->n_children); // union_flat.rs:817, intersection.rs:580
    if (ns->merged) {
        pl->d_bytes = ns->d_mbytes;
        pl->d_off_pos = ns->d_moff_pos;
        pl->d_off_len = ns->d_moff_len;
    }
    pl->nested = std::move(ns);
    return pl;
}
const uint32_t *II_ResultSet_DeviceDocIds(const II_ResultSet *rs) { return rs->d_docs; }
const double *II_ResultSet_DeviceScores(const II_ResultSet *rs) { return rs->d_scores; }

// ------------------------------------------------------------------------------------------------
// scoring
// ------------------------------------------------------------------------------------------------
double II_CalculateIDF(size_t total_docs, size_t term_docs) { // RS/idf/src/lib.rs:36-70
    if (term_docs == 0) term_docs = 1;
    const double value = 1.0 + (double)(total_docs + 1) / (double)term_docs;
    uint64_t bits;
    memcpy(&bits, &value, 8);
    return (double)((int)((bits >> 52) & 0x7FF) - 1023);
}
double II_CalculateIDF_BM25(size_t total_docs, size_t term_docs) { // :103-110
    total_docs = std::max(total_docs, term_docs);
    const double total = (double)total_docs, term = (double)term_docs;
    return std::log(1.0 + (total - term + 0.5) / (term + 0.5));
}

int II_Score(II_ResultSet *rs, II_Scorer scorer, const II_TermParams *terms, double agg_weight, const II_IndexStats *stats,
             const II_DocTable *docs, double min_score, uint64_t tanh_factor) {
    settle(rs);
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init() || !rs) return -1;
    if (rs->len == 0) {
        rs->scored = true;
        return 0;
    }
    if (!rs->has_freqs) return -1;
    cudaEventRecord(c.e0, c.stream);
    bool ok = true;
    if (scorer == II_SCORER_BM25 || scorer == II_SCORER_TFIDF || scorer == II_SCORER_TFIDF_DOCNORM)
        ok = ensure_slop(c, rs, nullptr, (uint32_t)rs->len);
    ok = ok && prepare_nested_scores(c, rs, scorer, stats, docs);
    const ScoreArgs sa = make_score_args(rs, scorer, terms, agg_weight, stats, docs, min_score, tanh_factor);
    ok = ok && ii_launch_score(sa, rs->d_docs, rs->d_freqs, rs->cap, nullptr, (uint32_t)rs->len, rs->d_scores, c.stream) == cudaSuccess;
    cudaEventRecord(c.e1, c.stream);
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    if (!ok) return -1;
    float ms = 0;
    cudaEventElapsedTime(&ms, c.e0, c.e1);
    c.stats.score_device_us = ms * 1000.0;
    c.stats.kernel_launches += 1;
    rs->scored = true;
    return 0;
}

// HAMMING (src/ext/default.c:475-497): the scorer looks at the query payload and the document payload only
int II_ScoreHamming(II_ResultSet *rs, const II_DocTable *docs, const void *qdata, size_t qdatalen) {
    settle(rs);
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init() || !rs) return -1;
    if (rs->len == 0) {
        rs->scored = true;
        return 0;
    }
    if (!docs || !docs->d_payload_off || qdatalen > 0xFFFFFFFFull) return -1;
    uint8_t *d_q = dalloc<uint8_t>(qdatalen ? qdatalen : 1);
    bool ok = d_q != nullptr;
    if (ok && qdatalen) ok = cudaMemcpyAsync(d_q, qdata, qdatalen, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
    cudaEventRecord(c.e0, c.stream);
    ok = ok && ii_launch_hamming(rs->d_docs, nullptr, (uint32_t)rs->len, docs->d_payloads, docs->d_payload_off, d_q, (uint32_t)qdatalen,
                                 rs->d_scores, c.stream) == cudaSuccess;
    cudaEventRecord(c.e1, c.stream);
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess; // also covers the pageable qdata copy
    dfree(d_q);
    if (!ok) return -1;
    float ms = 0;
    cudaEventElapsedTime(&ms, c.e0, c.e1);
    c.stats.score_device_us = ms * 1000.0;
    c.stats.kernel_launches += 1;
    rs->scored = true;
    return 0;
}

int II_ResultSet_Fetch(const II_ResultSet *rs, uint64_t *doc_ids, double *scores, uint32_t *child_freqs) {
    settle(rs);
    const size_t m = rs->len;
    if (m == 0) return 0;
    if (doc_ids) {
        std::vector<uint32_t> tmp(m);
        if (copy_sync(tmp.data(), rs->d_docs, m * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
        for (size_t i = 0; i < m; i++) doc_ids[i] = tmp[i];
    }
    if (scores) {
        if (rs->scored) {
            if (copy_sync(scores, rs->d_scores, m * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
        } else {
            for (size_t i = 0; i < m; i++) scores[i] = 0.0;
        }
    }
    if (child_freqs) {
        if (!rs->has_freqs) return -1;
        if (cudaMemcpy2DAsync(child_freqs, m * 4, rs->d_freqs, rs->cap * 4, m * 4, rs->n_children, cudaMemcpyDeviceToHost,
                              ctx().stream) != cudaSuccess ||
            cudaStreamSynchronize(ctx().stream) != cudaSuccess)
            return -1;
    }
    return 0;
}

size_t II_ResultSet_TopN(const II_ResultSet *rs, size_t n, uint64_t *doc_ids, double *scores) {
    settle(rs);
    Ctx &c = ctx();
    std::unique_lock<std::mutex> g(c.mu);
    if (!c.init() || rs->len == 0 || n == 0) return 0;
    const uint32_t k = (uint32_t)std::min<size_t>(n, rs->len);
    if (k > 1024) { // large LIMIT: download and partial-sort (rare; RPSorter heaps are offset+limit wide)
        g.unlock();
        std::vector<uint64_t> ids(rs->len);
        std::vector<double> sc(rs->len);
        if (II_ResultSet_Fetch(rs, ids.data(), sc.data(), nullptr) != 0) return 0;
        std::vector<uint32_t> idx(rs->len);
        for (size_t i = 0; i < rs->len; i++) idx[i] = (uint32_t)i;
        std::partial_sort(idx.begin(), idx.begin() + k, idx.end(), [&](uint32_t a, uint32_t b) {
            return sc[a] > sc[b] || (sc[a] == sc[b] && ids[a] < ids[b]);
        });
        for (uint32_t i = 0; i < k; i++) {
            doc_ids[i] = ids[idx[i]];
            scores[i] = sc[idx[i]];
        }
        return k;
    }
    const uint32_t lists = ii_topn_lists((uint32_t)rs->len);
    const size_t total = (size_t)lists * k;
    uint64_t *d_keys = dalloc<uint64_t>(total);
    uint32_t *d_ids = dalloc<uint32_t>(total);
    uint8_t *stg = c.stage(total * 12);
    bool ok = d_keys && d_ids && stg;
    uint64_t *h_keys = reinterpret_cast<uint64_t *>(stg);
    uint32_t *h_ids = reinterpret_cast<uint32_t *>(h_keys + total);
    ok = ok && ii_launch_topn(rs->d_docs, rs->d_scores, nullptr, (uint32_t)rs->len, k, d_keys, d_ids, c.stream) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(h_keys, d_keys, total * 8, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(h_ids, d_ids, total * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    dfree(d_keys);
    dfree(d_ids);
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    c.stats.kernel_launches += 1;
    if (!ok) return 0;
    return merge_topn_lists(h_keys, h_ids, total, k, doc_ids, scores);
}

// AND/OR -> score -> top-N with ONE host synchronisation: the hit count stays on the device, every
// kernel after the intersection reads it from rs->d_len.
size_t II_SearchTopN(II_PostingList *const *lists, size_t n, int is_union, II_Scorer scorer, const II_TermParams *terms,
                     double agg_weight, const II_IndexStats *stats, const II_DocTable *docs, size_t top_n, uint64_t *doc_ids,
                     double *scores, size_t *total_hits) {
    if (total_hits) *total_hits = 0;
    if (n == 0 || n > (size_t)(is_union ? kIIMaxUnionLists : kIIMaxLists) || top_n == 0) return 0;
    if (top_n > 1024) { // wide LIMITs take the unfused route
        II_ResultSet *rs = is_union ? II_Union(lists, n, 0) : II_Intersect(lists, n);
        if (!rs) return 0;
        if (total_hits) *total_hits = rs->len;
        size_t got = 0;
        if (II_Score(rs, scorer, terms, agg_weight, stats, docs, 0.0, 4) == 0) got = II_ResultSet_TopN(rs, top_n, doc_ids, scores);
        II_ResultSet_Free(rs);
        return got;
    }
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    if (!c.init()) return 0;
    PendingSearch p;
    if (!search_enqueue(c, lists, n, is_union, scorer, terms, agg_weight, stats, docs, top_n, p)) return 0;
    return search_finish(c, p, doc_ids, scores, total_hits);
}

// `nq` independent queries (one FT.SEARCH each) in one call.  AND queries with <= 8 terms and top_n <= 128 — the BASELINE
// shape — run FUSED: the whole batch is two kernel launches (membership + scorer + per-chunk top-N, then per-query top-N),
// one descriptor upload, one result download, one synchronisation.  Everything else (unions, wide ANDs, wide LIMITs) takes
// the per-query kernel chains, spread over a pool of streams.
namespace {
struct FusedScratch { // grow-only, owned by the batch entry point (serialised by its mutex)
    FusedQuery *h_q = nullptr, *d_q = nullptr;
    size_t q_cap = 0;
    uint64_t *d_cand_keys = nullptr, *d_out_keys = nullptr, *h_out_keys = nullptr;
    uint32_t *d_cand_ids = nullptr, *d_out_ids = nullptr, *h_out_ids = nullptr, *d_hits = nullptr, *h_hits = nullptr;
    uint32_t *d_item_q = nullptr; // work item -> query
    uint2 *d_win = nullptr;       // [items][kFusedMaxLists - 1] window of every other child per work item
    size_t cand_cap = 0, out_cap = 0, item_cap = 0;
    bool need(size_t nq, size_t cand, size_t out, size_t items) {
        if (items > item_cap) {
            cudaFree(d_item_q);
            cudaFree(d_win);
            d_item_q = nullptr;
            d_win = nullptr;
            item_cap = 0;
            const size_t cap = items + items / 4 + 1024;
            if (cudaMalloc(&d_item_q, cap * 4) != cudaSuccess || cudaMalloc(&d_win, cap * (kFusedMaxLists - 1) * sizeof(uint2)) != cudaSuccess)
                return false;
            item_cap = cap;
        }
        if (nq > q_cap) {
            cudaFreeHost(h_q);
            cudaFree(d_q);
            cudaFree(d_hits);
            cudaFreeHost(h_hits);
            h_q = d_q = nullptr;
            d_hits = h_hits = nullptr;
            q_cap = 0;
            const size_t cap = std::max<size_t>(nq, 1024);
            if (cudaMallocHost(&h_q, cap * sizeof(FusedQuery)) != cudaSuccess || cudaMalloc(&d_q, cap * sizeof(FusedQuery)) != cudaSuccess ||
                cudaMalloc(&d_hits, cap * 8) != cudaSuccess /* survivors + candidate fill */ || cudaMallocHost(&h_hits, cap * 4) != cudaSuccess)
                return false;
            q_cap = cap;
        }
        if (cand > cand_cap) {
            cudaFree(d_cand_keys);
            cudaFree(d_cand_ids);
            d_cand_keys = nullptr;
            d_cand_ids = nullptr;
            cand_cap = 0;
            const size_t cap = cand + cand / 4 + 4096;
            if (cudaMalloc(&d_cand_keys, cap * 8) != cudaSuccess || cudaMalloc(&d_cand_ids, cap * 4) != cudaSuccess) return false;
            cand_cap = cap;
        }
        if (out > out_cap) {
            cudaFree(d_out_keys);
            cudaFree(d_out_ids);
            cudaFreeHost(h_out_keys);
            cudaFreeHost(h_out_ids);
            d_out_keys = h_out_keys = nullptr;
            d_out_ids = h_out_ids = nullptr;
            out_cap = 0;
            const size_t cap = out + out / 4 + 4096;
            if (cudaMalloc(&d_out_keys, cap * 8) != cudaSuccess || cudaMalloc(&d_out_ids, cap * 4) != cudaSuccess ||
                cudaMallocHost(&h_out_keys, cap * 8) != cudaSuccess || cudaMallocHost(&h_out_ids, cap * 4) != cudaSuccess)
                return false;
            out_cap = cap;
        }
        return true;
    }
};

// Run the fusable queries idx[0..m) of the batch; false = nothing was written (the caller falls back to the chains)
bool fused_batch(Ctx &c, FusedScratch &fs, const std::vector<size_t> &idx, II_PostingList *const *const *lists, const size_t *n_lists,
                 II_Scorer scorer, const II_TermParams *const *terms, double agg_weight, const II_IndexStats *stats, const II_DocTable *docs,
                 size_t top_n, uint64_t *doc_ids, double *scores, size_t *counts, size_t *total_hits) {
    constexpr size_t kMaxCand = (size_t)96 << 20; // candidate slots per launch (x 12 B): larger batches are cut into several launches
    // aggregate child order of every query: stable sort ascending by num_estimated (intersection.rs:110-145).  The kernel drives
    // with child 0 of that order and scores the children in it, so the driver is not always the list with the fewest entries (a
    // field-mask filter keeps the unfiltered estimate, II_PostingList_FromBlocks): the scratch, the item count and the
    // candidate budget all come from the driver's length.
    std::vector<uint32_t> orders(idx.size() * kFusedMaxLists);
    std::vector<uint32_t> drive_chunks(idx.size());
    for (size_t k = 0; k < idx.size(); k++) {
        const size_t qi = idx[k];
        uint32_t *order = &orders[k * kFusedMaxLists];
        for (size_t t = 0; t < n_lists[qi]; t++) order[t] = (uint32_t)t;
        std::stable_sort(order, order + n_lists[qi], [&](uint32_t a, uint32_t b) { return lists[qi][a]->estimated < lists[qi][b]->estimated; });
        drive_chunks[k] = (uint32_t)((lists[qi][order[0]]->n + kIIChunk - 1) / kIIChunk);
    }
    size_t done = 0;
    while (done < idx.size()) {
        // sub-batch [done, stop): as many queries as fit the candidate budget
        size_t stop = done, items = 0;
        while (stop < idx.size()) {
            const size_t ch = drive_chunks[stop];
            if (stop > done && (items + ch) * top_n > kMaxCand) break;
            items += ch;
            stop++;
        }
        const size_t m = stop - done;
        if (!fs.need(m, items * top_n, m * top_n, items)) return false;
        uint32_t item0 = 0, max_children = 1;
        for (size_t k = 0; k < m; k++) {
            const size_t qi = idx[done + k];
            const size_t n = n_lists[qi];
            const uint32_t *order = &orders[(done + k) * kFusedMaxLists];
            FusedQuery &fq = fs.h_q[k];
            memset(&fq, 0, sizeof(fq));
            for (size_t t = 0; t < n; t++) {
                const II_PostingList *pl = lists[qi][order[t]];
                fq.ids[t] = pl->d_ids;
                fq.freqs[t] = pl->d_freqs;
                fq.len[t] = (uint32_t)pl->n;
                fq.weight[t] = terms[qi][order[t]].weight;
                fq.idf[t] = terms[qi][order[t]].idf;
                fq.bm25_idf[t] = terms[qi][order[t]].bm25_idf;
            }
            fq.n = (uint32_t)n;
            max_children = std::max(max_children, fq.n);
            fq.item0 = item0;
            fq.nchunks = drive_chunks[done + k];
            item0 += fq.nchunks;
        }
        // the kernels write item0 work items and item0 * top_n candidate slots.  item0 equals the `items` the scratch was sized
        // for just above; this is a backstop should the two sums ever diverge, not a path taken today
        if (item0 > fs.item_cap || (size_t)item0 * top_n > fs.cand_cap) return false;
        FusedCommon fc{};
        fc.scorer = (int)scorer;
        fc.agg_weight = agg_weight;
        fc.avg_doc_len = stats ? stats->avgDocLen : 0.0;
        fc.tanh_factor = 4;
        fc.doc_len = docs ? docs->d_len : nullptr;
        fc.doc_score = docs ? docs->d_score : nullptr;
        fc.max_freq = docs ? docs->d_maxf : nullptr;
        bool ok = cudaMemcpyAsync(fs.d_q, fs.h_q, m * sizeof(FusedQuery), cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
        cudaEventRecord(c.e0, c.stream);
        ok = ok && ii_launch_fused_search(fs.d_q, (uint32_t)m, item0, max_children, fc, (uint32_t)top_n, fs.d_item_q, fs.d_win, fs.d_cand_keys,
                                          fs.d_cand_ids, fs.d_hits, fs.d_out_keys, fs.d_out_ids, c.stream) == cudaSuccess;
        cudaEventRecord(c.e1, c.stream);
        ok = ok && cudaMemcpyAsync(fs.h_out_keys, fs.d_out_keys, m * top_n * 8, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(fs.h_out_ids, fs.d_out_ids, m * top_n * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(fs.h_hits, fs.d_hits, m * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
        if (!ok) {
            cudaGetLastError();
            return false;
        }
        float ms = 0;
        if (cudaEventElapsedTime(&ms, c.e0, c.e1) == cudaSuccess) c.stats.intersect_device_us += ms * 1000.0;
        c.stats.kernel_launches += 4;
        for (size_t k = 0; k < m; k++) {
            const size_t qi = idx[done + k];
            size_t w = 0;
            for (size_t t = 0; t < top_n; t++) {
                const uint32_t id = fs.h_out_ids[k * top_n + t];
                if (id == 0xFFFFFFFFu) break;
                doc_ids[qi * top_n + w] = id;
                uint64_t u = ~fs.h_out_keys[k * top_n + t];
                u = (u >> 63) ? (u & 0x7FFFFFFFFFFFFFFFull) : ~u;
                memcpy(&scores[qi * top_n + w], &u, 8);
                w++;
            }
            counts[qi] = w;
            if (total_hits) total_hits[qi] = fs.h_hits[k];
        }
        done = stop;
    }
    return true;
}
} // namespace

int II_SearchTopNBatch(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, int is_union, II_Scorer scorer,
                       const II_TermParams *const *terms, double agg_weight, const II_IndexStats *stats, const II_DocTable *docs,
                       size_t top_n, uint64_t *doc_ids, double *scores, size_t *counts, size_t *total_hits) {
    constexpr size_t kBatchSlots = 8;
    struct Pool {
        std::mutex mu;
        Ctx slot[kBatchSlots];
        FusedScratch fused;
    };
    static Pool pool;
    if (top_n == 0 || top_n > 1024) return -1;
    std::lock_guard<std::mutex> g(pool.mu);
    for (size_t i = 0; i < nq; i++) {
        counts[i] = 0;
        if (total_hits) total_hits[i] = 0;
    }
    // ---- fused path
    static const bool fused_on = [] {
        const char *e = getenv("II_B200_FUSED");
        return !(e && atoi(e) == 0);
    }();
    std::vector<size_t> fusable, rest;
    for (size_t i = 0; i < nq; i++) {
        if (n_lists[i] == 0 || n_lists[i] > (size_t)(is_union ? kIIMaxUnionLists : kIIMaxLists)) continue;
        bool empty = false;
        for (size_t t = 0; t < n_lists[i]; t++) empty |= lists[i][t]->n == 0;
        if (!is_union && empty) continue; // an empty child: the AND is empty (intersection.rs:363-417)
        // the legacy scorers divide by GetSlop, which walks term positions when the lists carry them: the per-query chain does
        bool wants_positions = false;
        if (scorer == II_SCORER_BM25 || scorer == II_SCORER_TFIDF || scorer == II_SCORER_TFIDF_DOCNORM)
            for (size_t t = 0; t < n_lists[i] && n_lists[i] > 1; t++) wants_positions |= lists[i][t]->d_off_len != nullptr;
        for (size_t t = 0; t < n_lists[i]; t++) wants_positions |= lists[i][t]->nested != nullptr; // nested sets: the chain recurses into them
        if (fused_on && !is_union && !wants_positions && n_lists[i] <= (size_t)kFusedMaxLists && top_n <= (size_t)kFusedMaxTopN)
            fusable.push_back(i);
        else
            rest.push_back(i);
    }
    if (!fusable.empty()) {
        double dev_us = 0;
        uint64_t launches = 0;
        {
            CtxScope scope(&pool.slot[0]);
            if (!pool.slot[0].init()) return -1;
            pool.slot[0].stats.intersect_device_us = 0;
            const uint64_t l0 = pool.slot[0].stats.kernel_launches;
            if (!fused_batch(pool.slot[0], pool.fused, fusable, lists, n_lists, scorer, terms, agg_weight, stats, docs, top_n, doc_ids, scores,
                             counts, total_hits))
                rest.insert(rest.end(), fusable.begin(), fusable.end());
            dev_us = pool.slot[0].stats.intersect_device_us;
            launches = pool.slot[0].stats.kernel_launches - l0;
        }
        // II_GetStats reports the calling thread's counters: device time of the fused launches (membership + scorer + top-N)
        ctx().stats.intersect_device_us = dev_us;
        ctx().stats.score_device_us = 0;
        ctx().stats.kernel_launches += launches;
    }
    // ---- per-query kernel chains on the stream pool: query i+1 is enqueued while query i runs, a slot is only
    // synchronised when it is needed again
    PendingSearch pend[kBatchSlots];
    size_t owner[kBatchSlots] = {0};
    uint64_t slot_launches0[kBatchSlots];
    for (size_t sl = 0; sl < kBatchSlots; sl++) slot_launches0[sl] = pool.slot[sl].stats.kernel_launches;
    auto finish = [&](size_t sl) {
        CtxScope scope(&pool.slot[sl]);
        const size_t qi = owner[sl];
        size_t tot = 0;
        counts[qi] = search_finish(pool.slot[sl], pend[sl], doc_ids + qi * top_n, scores + qi * top_n, &tot);
        if (total_hits) total_hits[qi] = tot;
    };
    int rc = 0;
    for (size_t r = 0; r < rest.size(); r++) {
        const size_t i = rest[r];
        const size_t sl = r % kBatchSlots;
        if (pend[sl].active) finish(sl);
        CtxScope scope(&pool.slot[sl]);
        if (!pool.slot[sl].init()) {
            rc = -1; // drain what is in flight before reporting the error: its buffers are freed in stream order
            break;
        }
        owner[sl] = i;
        search_enqueue(pool.slot[sl], lists[i], n_lists[i], is_union, scorer, terms[i], agg_weight, stats, docs, top_n, pend[sl]);
    }
    for (size_t sl = 0; sl < kBatchSlots; sl++)
        if (pend[sl].active) finish(sl);
    // the chains' launches, like the fused ones, go to the calling thread's counters
    for (size_t sl = 0; sl < kBatchSlots; sl++) ctx().stats.kernel_launches += pool.slot[sl].stats.kernel_launches - slot_launches0[sl];
    return rc;
}

// ------------------------------------------------------------------------------------------------
// term -> device posting list cache
// ------------------------------------------------------------------------------------------------
struct II_TermCache {
    struct Entry {
        uint64_t version = 0;
        II_PostingList *pl = nullptr;
        size_t refs = 0, bytes = 0;
        uint64_t tick = 0;
    };
    std::mutex mu;
    std::unordered_map<uint64_t, Entry> live;
    std::unordered_map<II_PostingList *, uint64_t> key_of;       // resident lists -> key
    std::unordered_map<II_PostingList *, size_t> zombies;        // replaced / invalidated while pinned: list -> refs left
    size_t max_bytes = 0, resident_bytes = 0;
    uint64_t tick = 0;
    bool keep_offsets = false; // Full-codec lists keep their term positions on the device (slop / in-order queries)
    II_TermCacheStats st{};
    void evict_locked() {
        while (resident_bytes > max_bytes) {
            uint64_t victim = 0, best = UINT64_MAX;
            bool found = false;
            for (auto &kv : live)
                if (kv.second.refs == 0 && kv.second.tick < best) {
                    best = kv.second.tick;
                    victim = kv.first;
                    found = true;
                }
            if (!found) break;
            Entry &e = live[victim];
            resident_bytes -= e.bytes;
            key_of.erase(e.pl);
            delete e.pl;
            live.erase(victim);
            st.evictions++;
        }
    }
    void drop_locked(uint64_t key) {
        auto it = live.find(key);
        if (it == live.end()) return;
        Entry &e = it->second;
        resident_bytes -= e.bytes;
        key_of.erase(e.pl);
        if (e.refs)
            zombies[e.pl] = e.refs; // still pinned by a running query: freed by the last Release
        else
            delete e.pl;
        live.erase(it);
    }
};

II_TermCache *II_TermCache_New(size_t max_device_bytes) {
    auto *c = new II_TermCache();
    c->max_bytes = max_device_bytes;
    return c;
}
void II_TermCache_Free(II_TermCache *c) {
    if (!c) return;
    for (auto &kv : c->live) delete kv.second.pl;
    for (auto &kv : c->zombies) delete kv.first;
    delete c;
}
void II_TermCache_KeepOffsets(II_TermCache *c, int on) {
    std::lock_guard<std::mutex> g(c->mu);
    c->keep_offsets = on != 0;
}
void II_TermCache_Invalidate(II_TermCache *c, uint64_t key) {
    std::lock_guard<std::mutex> g(c->mu);
    c->drop_locked(key);
}
II_TermCacheStats II_TermCache_GetStats(II_TermCache *c) {
    std::lock_guard<std::mutex> g(c->mu);
    II_TermCacheStats s = c->st;
    s.resident_bytes = c->resident_bytes;
    s.resident_lists = c->live.size();
    return s;
}

size_t II_TermCache_Acquire(II_TermCache *c, size_t n, const uint64_t *keys, const uint64_t *versions, const II_BlockView *const *blocks,
                            const size_t *nblocks, II_Codec codec, II_PostingList **out) {
    std::vector<size_t> miss;
    {
        std::lock_guard<std::mutex> g(c->mu);
        for (size_t i = 0; i < n; i++) {
            out[i] = nullptr;
            auto it = c->live.find(keys[i]);
            if (it != c->live.end() && it->second.version != versions[i]) { // the index was written / collected since
                c->drop_locked(keys[i]);
                it = c->live.end();
            }
            if (it != c->live.end()) {
                it->second.refs++;
                it->second.tick = ++c->tick;
                out[i] = it->second.pl;
                c->st.hits++;
            } else {
                miss.push_back(i);
            }
        }
    }
    if (!miss.empty()) {
        // the same key may appear twice among the misses (two queries of a batch sharing a term): decode it once
        std::vector<size_t> uniq;
        std::unordered_map<uint64_t, size_t> first_of;
        for (size_t i : miss)
            if (first_of.emplace(keys[i], uniq.size()).second) uniq.push_back(i);
        std::vector<const II_BlockView *> b(uniq.size());
        std::vector<size_t> nb(uniq.size());
        std::vector<II_PostingList *> built(uniq.size(), nullptr);
        for (size_t k = 0; k < uniq.size(); k++) {
            b[k] = blocks[uniq[k]];
            nb[k] = nblocks[uniq[k]];
        }
        bool keep;
        {
            std::lock_guard<std::mutex> g(c->mu);
            keep = c->keep_offsets;
        }
        from_blocks_batch(uniq.size(), b.data(), nb.data(), codec, keep, built.data());
        std::lock_guard<std::mutex> g(c->mu);
        for (size_t k = 0; k < uniq.size(); k++) {
            if (!built[k]) continue;
            const uint64_t key = keys[uniq[k]];
            c->drop_locked(key); // another thread may have inserted it meanwhile: ours replaces it
            II_TermCache::Entry e;
            e.version = versions[uniq[k]];
            e.pl = built[k];
            e.bytes = built[k]->n * 8;
            if (built[k]->d_off_len) { // + positions index + the encoded bytes that stay resident
                e.bytes += built[k]->n * 8;
                for (size_t x = 0; x < nb[k]; x++) e.bytes += b[k][x].len;
            }
            e.tick = ++c->tick;
            c->live[key] = e;
            c->key_of[built[k]] = key;
            c->resident_bytes += e.bytes;
            c->st.misses++;
        }
        for (size_t i : miss) {
            auto it = c->live.find(keys[i]);
            if (it == c->live.end()) continue;
            it->second.refs++;
            out[i] = it->second.pl;
        }
        c->evict_locked();
    }
    size_t got = 0;
    for (size_t i = 0; i < n; i++) got += out[i] != nullptr;
    return got;
}

void II_TermCache_Release(II_TermCache *c, size_t n, II_PostingList *const *lists) {
    std::lock_guard<std::mutex> g(c->mu);
    for (size_t i = 0; i < n; i++) {
        II_PostingList *pl = lists[i];
        if (!pl) continue;
        auto z = c->zombies.find(pl);
        if (z != c->zombies.end()) {
            if (--z->second == 0) {
                delete pl;
                c->zombies.erase(z);
            }
            continue;
        }
        auto k = c->key_of.find(pl);
        if (k == c->key_of.end()) continue;
        auto it = c->live.find(k->second);
        if (it != c->live.end() && it->second.refs) it->second.refs--;
    }
    c->evict_locked();
}

// ------------------------------------------------------------------------------------------------
// QueryIterator facade (src/iterators/iterator_api.h:46-151 contract)
// ------------------------------------------------------------------------------------------------
namespace {
// What an iterator over a finished result set walks on the host: its docIds, scores and per-hit freq (the sum of the children's),
// and the result it yields.  load() downloads a set; read / skip_to / rewind follow the QueryIterator contract on `b`.
struct HostCursor {
    II_IndexResult res;
    std::vector<uint64_t> ids;
    std::vector<double> scores; // zeros unless loaded with the set's scores
    std::vector<uint32_t> freq_sum; // empty: every hit yields freq 1
    size_t pos = 0; // index of the NEXT entry to yield
    bool load(const II_ResultSet *rs, bool with_scores) {
        const size_t m = rs->len;
        ids.resize(m);
        scores.assign(m, 0.0);
        if (II_ResultSet_Fetch(rs, ids.data(), with_scores ? scores.data() : nullptr, nullptr) != 0) return false;
        if (rs->has_freqs && m) {
            std::vector<uint32_t> fr((size_t)rs->n_children * m);
            if (II_ResultSet_Fetch(rs, nullptr, nullptr, fr.data()) != 0) return false;
            freq_sum.assign(m, 0);
            for (uint32_t ch = 0; ch < rs->n_children; ch++)
                for (size_t i = 0; i < m; i++) freq_sum[i] += fr[(size_t)ch * m + i];
        }
        return true;
    }
    static IteratorStatus eof(II_QueryIterator *b) {
        b->atEOF = true;
        b->current = nullptr;
        return ITERATOR_EOF;
    }
    void publish(II_QueryIterator *b, size_t i) {
        res.docId = ids[i];
        res.freq = freq_sum.empty() ? 1u : freq_sum[i];
        res.data.metric = scores[i];
        b->lastDocId = ids[i];
        b->current = &res;
    }
    IteratorStatus read(II_QueryIterator *b) {
        if (pos >= ids.size()) return eof(b);
        publish(b, pos++);
        return ITERATOR_OK;
    }
    IteratorStatus skip_to(II_QueryIterator *b, t_docId doc) {
        auto lb = std::lower_bound(ids.begin() + pos, ids.end(), doc);
        if (lb == ids.end()) {
            pos = ids.size();
            return eof(b);
        }
        const size_t i = (size_t)(lb - ids.begin());
        publish(b, i);
        pos = i + 1;
        return *lb == doc ? ITERATOR_OK : ITERATOR_NOTFOUND;
    }
    void rewind(II_QueryIterator *b) {
        pos = 0;
        b->atEOF = false;
        b->lastDocId = 0;
        b->current = nullptr;
    }
};

struct ResultIter {
    II_QueryIterator base; // MUST be first: RediSearch sees a QueryIterator*
    HostCursor cur;
};
inline ResultIter *RI(II_QueryIterator *b) { return reinterpret_cast<ResultIter *>(b); }

size_t ri_num_estimated(const II_QueryIterator *b) { return reinterpret_cast<const ResultIter *>(b)->cur.ids.size(); }
IteratorStatus ri_read(II_QueryIterator *b) { return RI(b)->cur.read(b); }
IteratorStatus ri_skip_to(II_QueryIterator *b, t_docId doc) { return RI(b)->cur.skip_to(b, doc); }
ValidateStatus ri_revalidate(II_QueryIterator *, struct IndexSpec *) { return VALIDATE_OK; } // a snapshot never moves
void ri_rewind(II_QueryIterator *b) { RI(b)->cur.rewind(b); }
void ri_free(II_QueryIterator *b) { delete RI(b); }
} // namespace

II_QueryIterator *II_NewResultIterator(II_ResultSet *rs, double weight) {
    settle(rs);
    if (!rs) return nullptr;
    auto *it = new ResultIter();
    memset(&it->base, 0, sizeof(it->base));
    memset(&it->cur.res, 0, sizeof(it->cur.res));
    const bool ok = it->cur.load(rs, true);
    it->base.type = rs->is_union ? II_IteratorType_Union : II_IteratorType_Intersect;
    it->base.NumEstimated = ri_num_estimated;
    it->base.Read = ri_read;
    it->base.SkipTo = ri_skip_to;
    it->base.Revalidate = ri_revalidate;
    it->base.Free = ri_free;
    it->base.Rewind = ri_rewind;
    it->cur.res.data.tag = II_ResultData_Metric;
    it->cur.res.weight = weight;
    it->cur.res.fieldMask = ~(unsigned __int128)0; // RS_FIELDMASK_ALL
    II_ResultSet_Free(rs);
    if (!ok) {
        delete it;
        return nullptr;
    }
    return &it->base;
}

// ------------------------------------------------------------------------------------------------
// The reference's iterator constructors (RS/headers/iterators_ffi.h:309,594) and scorer extension entry point
// (src/extension.c:121-145, src/redisearch.h:277-287) on top of the device algebra.
//
// Children may be (a) our own iterators — term leaves (II_NewTermIterator*), NOT / OPTIONAL wrappers, results of a nested
// AND / OR built here — which stay on the device, or (b) FOREIGN iterators (anything with the QueryIterator vtable: numeric,
// tag, geo ... leaves of RediSearch): those are drained through Read() once, their docIds / freqs uploaded, and take part
// as one more device list.  The iterator tree is evaluated eagerly at construction (a few kernels + one synchronisation);
// the returned iterator walks the finished result set and carries, in `current`, the back-pointer the registered scoring
// functions need to return a score computed ON THE DEVICE for the whole result set at the first call.
// ------------------------------------------------------------------------------------------------
namespace {
constexpr uint64_t kNodeMagic = 0xB200D15C0FFEE5ull;
const II_DocTable *g_default_docs = nullptr;

enum NodeKind { NODE_LEAF = 0, NODE_RESULT = 1, NODE_EMPTY = 2, NODE_WILDCARD = 3 };
enum LeafMode { LEAF_REQUIRED = 0, LEAF_NOT = 1, LEAF_OPTIONAL = 2 };

struct NodeIter {
    II_QueryIterator base; // MUST be first
    uint64_t magic = kNodeMagic;
    NodeKind kind = NODE_EMPTY;
    // leaf
    II_PostingList *pl = nullptr;
    bool owns_pl = false;
    II_TermCache *cache = nullptr; // non-NULL: pl is pinned in this cache (released, not freed)
    II_TermParams term{1.0, 0.0, 0.0};
    LeafMode mode = LEAF_REQUIRED;
    void *host_term = nullptr;               // the host's RSQueryTerm (NewInvIndIterator_TermQuery): owned, released with
    void (*host_term_free)(void *) = nullptr; // the host's Term_Free
    uint64_t max_doc_id = 0; // NOT / OPTIONAL: the universe is 1..max_doc_id; wildcard: top_id
    bool past_end = false;   // wildcard: a read / skip found nothing (wildcard.rs `past_end`)
    // result of an evaluated AND / OR (or a leaf that is read directly)
    II_ResultSet *rs = nullptr;
    std::vector<II_TermParams> terms; // per child, in the order of the constructor's `its`
    std::vector<std::string> term_strs; // per child: the term's text where the host gave one (EXPLAINSCORE)
    std::string term_str;               // leaf: QueryTerm_GetStrAndLen of host_term
    double agg_weight = 1.0;
    int scored_with = -1; // II_Scorer the host score array holds
    const II_DocTable *docs = nullptr;
    bool host_ready = false; // cur holds rs
    HostCursor cur;
    ~NodeIter() {
        if (host_term && host_term_free) host_term_free(host_term);
        if (pl) {
            if (cache)
                II_TermCache_Release(cache, 1, &pl);
            else if (owns_pl)
                delete pl;
        }
        delete rs;
    }
};
inline NodeIter *NI(II_QueryIterator *b) { return reinterpret_cast<NodeIter *>(b); }
inline bool is_node(const II_QueryIterator *b) { return b && reinterpret_cast<const NodeIter *>(b)->magic == kNodeMagic && b->Free != nullptr; }

void host_free(void *p) { // `its` arrays come from the Redis allocator
    static void (**rm_free)(void *) = reinterpret_cast<void (**)(void *)>(dlsym(RTLD_DEFAULT, "RedisModule_Free"));
    if (rm_free && *rm_free)
        (*rm_free)(p);
    else
        free(p);
}

void *host_alloc(size_t n) { // what the host frees with rm_free must come from the Redis allocator
    static void *(**rm_alloc)(size_t) = reinterpret_cast<void *(**)(size_t)>(dlsym(RTLD_DEFAULT, "RedisModule_Alloc"));
    return (rm_alloc && *rm_alloc) ? (*rm_alloc)(n) : malloc(n);
}

// a leaf that is read directly (single-term query: the reducers hand the child back) becomes a 1-child result
bool node_materialise(NodeIter *it) {
    if (it->kind == NODE_LEAF && !it->rs) {
        II_PostingList *one[1] = {it->pl};
        it->rs = II_Union(one, 1, 0);
        if (!it->rs) return false;
        it->terms.assign(1, it->term);
        it->term_strs.assign(1, it->term_str);
        it->agg_weight = 1.0;
    }
    return true;
}
bool node_host(NodeIter *it) {
    if (it->host_ready) return true;
    if (it->kind == NODE_EMPTY) {
        it->host_ready = true;
        return true;
    }
    if (!node_materialise(it) || !it->rs || !it->cur.load(it->rs, false)) return false;
    it->host_ready = true;
    return true;
}
size_t node_num_estimated(const II_QueryIterator *b) {
    const NodeIter *it = reinterpret_cast<const NodeIter *>(b);
    if (it->kind == NODE_EMPTY) return 0;
    if (it->rs) return it->kind == NODE_RESULT ? it->rs->estimated : it->rs->len; // AND: min over the children, OR: their sum
    if (it->mode != LEAF_REQUIRED) return (size_t)it->max_doc_id; // not.rs / optional.rs num_estimated = max_doc_id
    return it->pl ? it->pl->estimated : 0;
}
IteratorStatus node_read(II_QueryIterator *b) {
    NodeIter *it = NI(b);
    return node_host(it) ? it->cur.read(b) : HostCursor::eof(b);
}
IteratorStatus node_skip_to(II_QueryIterator *b, t_docId doc) {
    NodeIter *it = NI(b);
    return node_host(it) ? it->cur.skip_to(b, doc) : HostCursor::eof(b);
}
ValidateStatus node_revalidate(II_QueryIterator *, struct IndexSpec *) { return VALIDATE_OK; } // a snapshot never moves
void node_rewind(II_QueryIterator *b) { NI(b)->cur.rewind(b); }
void node_free(II_QueryIterator *b) { delete NI(b); }

// ---- wildcard (rqe_iterators/src/wildcard.rs:83-180): a counter over 1..top_id yielding one virtual result
size_t wc_num_estimated(const II_QueryIterator *b) { return (size_t) reinterpret_cast<const NodeIter *>(b)->max_doc_id; }
bool wc_exhausted(NodeIter *it) {
    if (it->past_end || it->base.lastDocId >= it->max_doc_id) {
        it->past_end = true;
        it->base.atEOF = true;
        it->base.current = nullptr;
        return true;
    }
    return false;
}
IteratorStatus wc_read(II_QueryIterator *b) {
    NodeIter *it = NI(b);
    if (wc_exhausted(it)) return ITERATOR_EOF;
    b->lastDocId += 1;
    it->cur.res.docId = b->lastDocId;
    b->current = &it->cur.res;
    return ITERATOR_OK;
}
IteratorStatus wc_skip_to(II_QueryIterator *b, t_docId doc) {
    NodeIter *it = NI(b);
    if (wc_exhausted(it)) return ITERATOR_EOF;
    if (doc > it->max_doc_id) { // beyond the last document: the position stays where the last yield left it
        it->past_end = true;
        b->atEOF = true;
        b->current = nullptr;
        return ITERATOR_EOF;
    }
    b->lastDocId = doc;
    it->cur.res.docId = doc;
    b->current = &it->cur.res;
    return ITERATOR_OK;
}
void wc_rewind(II_QueryIterator *b) {
    NodeIter *it = NI(b);
    it->past_end = false;
    b->atEOF = false;
    b->lastDocId = 0;
    b->current = nullptr;
}

NodeIter *new_node(NodeKind kind, uint32_t type, double weight) {
    auto *it = new NodeIter();
    memset(&it->base, 0, sizeof(it->base));
    memset(&it->cur.res, 0, sizeof(it->cur.res));
    it->kind = kind;
    it->base.type = type;
    it->base.NumEstimated = node_num_estimated;
    it->base.Read = node_read;
    it->base.SkipTo = node_skip_to;
    it->base.Revalidate = node_revalidate;
    it->base.Free = node_free;
    it->base.Rewind = node_rewind;
    it->cur.res.data.tag = II_ResultData_Metric;
    it->cur.res.weight = weight;
    it->cur.res.fieldMask = ~(unsigned __int128)0; // RS_FIELDMASK_ALL
    // back-pointer for the scoring functions: bytes the Metric variant of the reference's result union does not use
    memcpy(it->cur.res.data._rest, &kNodeMagic, 8);
    NodeIter *self = it;
    memcpy(it->cur.res.data._rest + 8, &self, 8);
    it->docs = g_default_docs;
    if (kind == NODE_EMPTY) it->base.atEOF = false;
    return it;
}

// a FOREIGN iterator -> device posting list (docIds ascending as the contract guarantees; freq = current->freq)
II_PostingList *drain_foreign(II_QueryIterator *f, uint8_t *tag, double *weight) {
    std::vector<uint64_t> ids;
    std::vector<uint32_t> freqs;
    if (f->Rewind) f->Rewind(f);
    bool first = true;
    while (f->Read(f) == ITERATOR_OK) {
        ids.push_back(f->lastDocId);
        freqs.push_back(f->current ? f->current->freq : 1u);
        if (first && f->current) { // what kind of result the child yields, and its weight (the scorers treat the kinds differently)
            *tag = (uint8_t)f->current->data.tag;
            *weight = f->current->weight;
            first = false;
        }
    }
    return II_PostingList_FromArrays(ids.data(), freqs.data(), ids.size());
}

struct ChildView { // what the algebra needs from a child
    II_PostingList *pl = nullptr;
    bool temp = false; // built here (foreign / nested result): freed after the evaluation
    LeafMode mode = LEAF_REQUIRED;
    II_TermParams term{1.0, 1.0, 1.0};
    std::string str;
};
bool child_view(II_QueryIterator *c, ChildView &v, bool need_offsets) {
    if (is_node(c)) {
        NodeIter *n = NI(c);
        if (n->kind == NODE_LEAF) {
            v.pl = n->pl;
            v.mode = n->mode;
            v.term = n->term;
            v.str = n->term_str;
            if (v.pl && v.pl->nested && v.pl->nested->term_strs.empty()) v.pl->nested->term_strs = n->term_strs; // -(a|b), ~(a b)
            return v.pl != nullptr;
        }
        if (n->kind == NODE_WILDCARD) { // every document, as a virtual result with freq 1: a leaf with idf = 1 scores the same
            v.pl = posting_list_all_docs(n->max_doc_id);
            v.temp = true;
            v.term = II_TermParams{n->cur.res.weight, 1.0, 1.0};
            return v.pl != nullptr;
        }
        if (n->kind == NODE_RESULT && n->rs) {
            // nested AND / OR: stays on the device as one child (the scorers recurse into it, its term positions are merged);
            // the child node gives its result set away
            if (n->rs->has_freqs && n->rs->n_children <= (uint32_t)kIIMaxLists && !n->host_ready) {
                II_ResultSet *inner = n->rs;
                n->rs = nullptr;
                v.pl = II_ResultSet_IntoChild(inner, n->terms.data(), n->agg_weight, need_offsets ? 1 : 0);
                if (v.pl && v.pl->nested) v.pl->nested->term_strs = n->term_strs;
                v.temp = true;
                v.term = II_TermParams{n->agg_weight, 1.0, 1.0}; // not read: the nested set carries its own
                return v.pl != nullptr;
            }
            if (need_offsets) return false;
            // a quick union (no per-child freqs: never scored): its docIds as a flat list
            if (!node_host(n)) return false;
            std::vector<uint32_t> fr(n->cur.ids.size(), 1u);
            for (size_t i = 0; i < fr.size() && i < n->cur.freq_sum.size(); i++) fr[i] = n->cur.freq_sum[i];
            v.pl = II_PostingList_FromArrays(n->cur.ids.data(), fr.data(), n->cur.ids.size());
            v.temp = true;
            v.term = II_TermParams{n->agg_weight, 1.0, 1.0};
            if (v.pl) v.pl->result_tag = n->rs->is_union ? 1 : 2;
            return v.pl != nullptr;
        }
        return false;
    }
    if (need_offsets) return false;
    uint8_t tag = 8;
    double w = 1.0;
    v.pl = drain_foreign(c, &tag, &w);
    v.temp = true;
    if (v.pl) v.pl->result_tag = tag;
    // a numeric / metric result is an "irrelevant token" for BM25STD (default.c:296-300) and weight * freq for TFIDF (:104)
    v.term = II_TermParams{w, 1.0, (tag == 16 || tag == 32) ? 0.0 : 1.0};
    return v.pl != nullptr;
}
bool child_is_empty(const II_QueryIterator *c) {
    if (!c) return true;
    if (c->type == II_IteratorType_Empty) return true;
    if (is_node(c)) {
        const NodeIter *n = reinterpret_cast<const NodeIter *>(c);
        if (n->kind == NODE_EMPTY) return true;
        if (n->kind == NODE_LEAF && n->mode == LEAF_REQUIRED && n->pl && n->pl->n == 0) return true;
        if (n->kind == NODE_RESULT && n->rs && n->rs->len == 0) return true;
    }
    return false;
}
} // namespace

void II_SetDefaultDocTable(const II_DocTable *docs) { g_default_docs = docs; }

II_QueryIterator *II_NewEmptyIterator(void) { return &new_node(NODE_EMPTY, II_IteratorType_Empty, 1.0)->base; }

// NewWildcardIterator_NonOptimized (RS/headers/iterators_ffi.h; rqe_iterators/src/wildcard.rs:83-96): every docId 1..top_id as a
// VIRTUAL result with freq 1, field mask ALL and the given weight.  As a child of our AND it is stripped, as a child of a quick
// union it becomes the union (union_reducer.rs:41-53), in a full union / under NOT / OPTIONAL it takes part as the device list
// 1..top_id.
II_QueryIterator *II_NewWildcardIterator(t_docId top_id, double weight) {
    NodeIter *n = new_node(NODE_WILDCARD, II_IteratorType_Wildcard, weight);
    n->max_doc_id = top_id;
    n->base.NumEstimated = wc_num_estimated;
    n->base.Read = wc_read;
    n->base.SkipTo = wc_skip_to;
    n->base.Rewind = wc_rewind;
    n->cur.res.data.tag = II_ResultData_Virtual;
    memset(n->cur.res.data._rest, 0, sizeof(n->cur.res.data._rest)); // a virtual result carries no payload (and no scorer back-pointer)
    n->cur.res.freq = 1;
    return &n->base;
}
// the reference's own name and signature (RS/headers/iterators_ffi.h:647)
II_QueryIterator *NewWildcardIterator_NonOptimized(t_docId max_id, double weight) { return II_NewWildcardIterator(max_id, weight); }

II_QueryIterator *II_NewTermIterator(II_PostingList *pl, int take_ownership, double weight, double idf, double bm25_idf) {
    if (!pl) return nullptr;
    NodeIter *it = new_node(NODE_LEAF, 1 /* IteratorType_InvIdxTerm */, weight);
    it->pl = pl;
    it->owns_pl = take_ownership != 0;
    it->term = II_TermParams{weight, idf, bm25_idf};
    return &it->base;
}

// Term leaf straight from the host's InvertedIndex: the block accessors of RS/headers/inverted_index_ffi.h:102-132,286,387,425,444
// are resolved in the host process at first use (+ IndexBlock_DataLen, the one accessor the FFI does not have yet — three lines
// of Rust, INTEGRATION.md §2).  With a cache the decoded list is shared between queries and revalidated by
// (gc_marker, num_entries).
II_QueryIterator *II_NewTermIterator_FromIndex(const void *inverted_index, II_Codec codec, double weight, double idf, double bm25_idf,
                                               II_TermCache *cache) {
    struct Api {
        size_t (*NumBlocks)(const void *) = nullptr;
        const void *(*BlockRef)(const void *, size_t) = nullptr;
        const char *(*Data)(const void *) = nullptr;
        size_t (*DataLen)(const void *) = nullptr;
        uint64_t (*FirstId)(const void *) = nullptr;
        uint64_t (*LastId)(const void *) = nullptr;
        uint16_t (*NumEntries)(const void *) = nullptr;
        uint32_t (*GcMarker)(const void *) = nullptr;
        size_t (*IndexEntries)(const void *) = nullptr;
        bool ok = false;
    };
    static Api api = [] {
        Api a;
        a.NumBlocks = reinterpret_cast<decltype(a.NumBlocks)>(dlsym(RTLD_DEFAULT, "InvertedIndex_NumBlocks"));
        a.BlockRef = reinterpret_cast<decltype(a.BlockRef)>(dlsym(RTLD_DEFAULT, "InvertedIndex_BlockRef"));
        a.Data = reinterpret_cast<decltype(a.Data)>(dlsym(RTLD_DEFAULT, "IndexBlock_Data"));
        a.DataLen = reinterpret_cast<decltype(a.DataLen)>(dlsym(RTLD_DEFAULT, "IndexBlock_DataLen"));
        a.FirstId = reinterpret_cast<decltype(a.FirstId)>(dlsym(RTLD_DEFAULT, "IndexBlock_FirstId"));
        a.LastId = reinterpret_cast<decltype(a.LastId)>(dlsym(RTLD_DEFAULT, "IndexBlock_LastId"));
        a.NumEntries = reinterpret_cast<decltype(a.NumEntries)>(dlsym(RTLD_DEFAULT, "IndexBlock_NumEntries"));
        a.GcMarker = reinterpret_cast<decltype(a.GcMarker)>(dlsym(RTLD_DEFAULT, "InvertedIndex_GcMarker"));
        a.IndexEntries = reinterpret_cast<decltype(a.IndexEntries)>(dlsym(RTLD_DEFAULT, "InvertedIndex_NumEntries"));
        a.ok = a.NumBlocks && a.BlockRef && a.Data && a.DataLen && a.FirstId && a.LastId && a.NumEntries;
        return a;
    }();
    if (!api.ok || !inverted_index) {
        fprintf(stderr, "ii_b200: the host process does not export the InvertedIndex block accessors (inverted_index_ffi.h + IndexBlock_DataLen)\n");
        return nullptr;
    }
    const size_t nb = api.NumBlocks(inverted_index);
    std::vector<II_BlockView> views(nb);
    for (size_t b = 0; b < nb; b++) {
        const void *blk = api.BlockRef(inverted_index, b);
        views[b] = II_BlockView{api.FirstId(blk), api.LastId(blk), api.NumEntries(blk), reinterpret_cast<const uint8_t *>(api.Data(blk)), api.DataLen(blk)};
    }
    II_PostingList *pl = nullptr;
    if (cache) {
        const uint64_t key = (uint64_t)(uintptr_t)inverted_index;
        const uint64_t version = ((uint64_t)(api.GcMarker ? api.GcMarker(inverted_index) : 0) << 32) ^ (uint64_t)(api.IndexEntries ? api.IndexEntries(inverted_index) : nb);
        const II_BlockView *bl[1] = {views.data()};
        const size_t nbs[1] = {nb};
        II_TermCache_Acquire(cache, 1, &key, &version, bl, nbs, codec, &pl);
    } else {
        pl = II_PostingList_FromBlocks(views.data(), nb, codec, 0, 1);
    }
    if (!pl) return nullptr;
    II_QueryIterator *it = II_NewTermIterator(pl, cache ? 0 : 1, weight, idf, bm25_idf);
    if (it && cache) NI(it)->cache = cache;
    return it;
}

// ---- the term leaf with the reference's OWN name and signature (RS/headers/iterators_ffi.h:404) ---------------------------
// What Term::new does (RS/rqe_iterators/src/inverted_index/term.rs:77-100) with what the host process exports:
//   codec        <- InvertedIndex_Flags(idx) & INDEX_STORAGE_MASK   (the table of NewInvertedIndex_Ex,
//                   RS/c_entrypoint/inverted_index_ffi/src/lib.rs:49-165; II_CodecFromIndexFlags)
//   total_docs   <- IndexSpec_GetStats(sctx->spec, &stats).numDocs  (src/spec.c:1830; RedisSearchCtx = {redisCtx, spec, ...},
//                   src/search_ctx.h:60-64)
//   term_docs    <- InvertedIndex_NumDocs(idx)                      (unique docs, inverted_index_ffi.h:434)
//   the IDFs are computed (RS/idf/src/lib.rs) and stored into the term with QueryTerm_SetIDFs so that the host's scorers see
//   them too; the term is owned by the iterator and released with Term_Free.
// The field-mask filter of the Mask variant is applied at decode time (FilterMaskReader); the Index variant only selects
// field-expiration checks, which this library does not do.  NULL (nothing consumed, the term still the caller's) when the host
// does not export an accessor, or the index cannot be represented: the caller keeps the reference's iterator.
namespace {
II_TermCache *g_default_cache = nullptr;
int g_raw_docid_encoding = 0;
struct RSIndexStatsHost { // src/redisearch.h:245-249
    size_t numDocs, numTerms;
    double avgDocLen;
};
} // namespace
void II_SetDefaultTermCache(II_TermCache *cache) { g_default_cache = cache; }
void II_SetRawDocIdEncoding(int raw) { g_raw_docid_encoding = raw; }
int II_CodecFromIndexFlags(uint32_t flags, int raw_doc_id_encoding) {
    constexpr uint32_t kOffsets = 0x01, kFields = 0x02, kFreqs = 0x10, kNumeric = 0x20, kWide = 0x80; // src/spec.h:171-181
    switch (flags & (kOffsets | kFields | kFreqs | kNumeric | kWide)) {
    case kFreqs | kOffsets | kFields: return II_CODEC_FULL;
    case kFreqs | kOffsets | kFields | kWide: return II_CODEC_FULL_WIDE;
    case kFreqs | kFields: return II_CODEC_FREQS_FIELDS;
    case kFreqs | kFields | kWide: return II_CODEC_FREQS_FIELDS_WIDE;
    case kFreqs: return II_CODEC_FREQS_ONLY;
    case kFields: return II_CODEC_FIELDS_ONLY;
    case kFields | kWide: return II_CODEC_FIELDS_ONLY_WIDE;
    case kFields | kOffsets: return II_CODEC_FIELDS_OFFSETS;
    case kFields | kOffsets | kWide: return II_CODEC_FIELDS_OFFSETS_WIDE;
    case kOffsets: return II_CODEC_OFFSETS_ONLY;
    case kFreqs | kOffsets: return II_CODEC_FREQS_OFFSETS;
    case 0: return raw_doc_id_encoding ? II_CODEC_RAW_DOCIDS_ONLY : II_CODEC_DOCIDS_ONLY;
    default: return -1; // numeric (II_NumericList_*) or a combination NewInvertedIndex_Ex panics on
    }
}
II_QueryIterator *NewInvIndIterator_TermQuery(const void *idx, const void *sctx, II_FieldMaskOrIndex field_mask_or_index, void *term,
                                              double weight) {
    struct Api {
        uint32_t (*Flags)(const void *) = nullptr;
        uint32_t (*NumDocs)(const void *) = nullptr;
        void (*GetStats)(void *, RSIndexStatsHost *) = nullptr;
        void (*SetIDFs)(void *, double, double) = nullptr;
        void (*TermFree)(void *) = nullptr;
        bool ok = false;
    };
    static Api api = [] {
        Api a;
        a.Flags = reinterpret_cast<decltype(a.Flags)>(dlsym(RTLD_DEFAULT, "InvertedIndex_Flags"));
        a.NumDocs = reinterpret_cast<decltype(a.NumDocs)>(dlsym(RTLD_DEFAULT, "InvertedIndex_NumDocs"));
        a.GetStats = reinterpret_cast<decltype(a.GetStats)>(dlsym(RTLD_DEFAULT, "IndexSpec_GetStats"));
        a.SetIDFs = reinterpret_cast<decltype(a.SetIDFs)>(dlsym(RTLD_DEFAULT, "QueryTerm_SetIDFs"));
        a.TermFree = reinterpret_cast<decltype(a.TermFree)>(dlsym(RTLD_DEFAULT, "Term_Free"));
        a.ok = a.Flags && a.NumDocs && a.GetStats && a.SetIDFs && a.TermFree;
        return a;
    }();
    if (!api.ok || !idx || !sctx || !term) return nullptr;
    const int codec = II_CodecFromIndexFlags(api.Flags(idx), g_raw_docid_encoding);
    if (codec < 0) return nullptr;
    void *spec = static_cast<void *const *>(sctx)[1];
    if (!spec) return nullptr;
    RSIndexStatsHost st{};
    api.GetStats(spec, &st);
    const size_t term_docs = api.NumDocs(idx);
    const double idf = II_CalculateIDF(st.numDocs, term_docs), bm25_idf = II_CalculateIDF_BM25(st.numDocs, term_docs);
    II_QueryIterator *it = nullptr;
    const bool masked = field_mask_or_index.tag == 1 /* FieldMaskOrIndex_Mask */ && ~field_mask_or_index.mask != 0 /* not RS_FIELDMASK_ALL */ &&
                        ii_codec_has_mask(codec);
    if (!masked) {
        it = II_NewTermIterator_FromIndex(idx, (II_Codec)codec, weight, idf, bm25_idf, g_default_cache);
    } else { // FilterMaskReader: decode with the filter (not cached: the cache holds unfiltered lists)
        struct BlockApi {
            size_t (*NumBlocks)(const void *) = nullptr;
            const void *(*BlockRef)(const void *, size_t) = nullptr;
            const char *(*Data)(const void *) = nullptr;
            size_t (*DataLen)(const void *) = nullptr;
            uint64_t (*FirstId)(const void *) = nullptr;
            uint64_t (*LastId)(const void *) = nullptr;
            uint16_t (*NumEntries)(const void *) = nullptr;
        } b;
        b.NumBlocks = reinterpret_cast<decltype(b.NumBlocks)>(dlsym(RTLD_DEFAULT, "InvertedIndex_NumBlocks"));
        b.BlockRef = reinterpret_cast<decltype(b.BlockRef)>(dlsym(RTLD_DEFAULT, "InvertedIndex_BlockRef"));
        b.Data = reinterpret_cast<decltype(b.Data)>(dlsym(RTLD_DEFAULT, "IndexBlock_Data"));
        b.DataLen = reinterpret_cast<decltype(b.DataLen)>(dlsym(RTLD_DEFAULT, "IndexBlock_DataLen"));
        b.FirstId = reinterpret_cast<decltype(b.FirstId)>(dlsym(RTLD_DEFAULT, "IndexBlock_FirstId"));
        b.LastId = reinterpret_cast<decltype(b.LastId)>(dlsym(RTLD_DEFAULT, "IndexBlock_LastId"));
        b.NumEntries = reinterpret_cast<decltype(b.NumEntries)>(dlsym(RTLD_DEFAULT, "IndexBlock_NumEntries"));
        if (!(b.NumBlocks && b.BlockRef && b.Data && b.DataLen && b.FirstId && b.LastId && b.NumEntries)) return nullptr;
        const size_t nb = b.NumBlocks(idx);
        std::vector<II_BlockView> views(nb);
        for (size_t i = 0; i < nb; i++) {
            const void *blk = b.BlockRef(idx, i);
            views[i] = II_BlockView{b.FirstId(blk), b.LastId(blk), b.NumEntries(blk), reinterpret_cast<const uint8_t *>(b.Data(blk)), b.DataLen(blk)};
        }
        const uint64_t f128[2] = {(uint64_t)field_mask_or_index.mask, (uint64_t)(field_mask_or_index.mask >> 64)};
        II_PostingList *pl = nullptr;
        if (ii_codec_is_wide(codec)) {
            pl = II_PostingList_FromBlocksWideMask(views.data(), nb, (II_Codec)codec, f128, 1);
        } else if ((uint32_t)f128[0] == 0) {
            it = II_NewEmptyIterator(); // a 32-bit-mask index cannot meet a filter whose low 32 bits are clear
        } else {
            pl = II_PostingList_FromBlocks(views.data(), nb, (II_Codec)codec, (uint32_t)f128[0], 1);
        }
        if (pl) it = II_NewTermIterator(pl, 1, weight, idf, bm25_idf);
    }
    if (!it) return nullptr;
    api.SetIDFs(term, idf, bm25_idf);
    {
        static const char *(*get_str)(const void *, size_t *) =
            reinterpret_cast<const char *(*)(const void *, size_t *)>(dlsym(RTLD_DEFAULT, "QueryTerm_GetStrAndLen"));
        size_t len = 0;
        const char *str = get_str ? get_str(term, &len) : nullptr;
        if (str && is_node(it)) NI(it)->term_str.assign(str, len);
    }
    NI(it)->host_term = term;
    NI(it)->host_term_free = api.TermFree;
    if (it->type != II_IteratorType_Empty) it->type = 1; // IteratorType_InvIdxTerm
    return it;
}

// `-(a|b)`, `~(a b)`: an evaluated nested AND / OR under NOT / OPTIONAL becomes a leaf whose list is the nested set's view
// (II_ResultSet_IntoChild): excluded docIds for NOT; for OPTIONAL the set's recursive score where it matches, with the OPTIONAL's
// weight as the aggregate's own (optional.rs:260,302 `real.weight = self.weight`).  false: not convertible (the node is untouched,
// or — when the device refused the view — left empty).
static bool nested_node_to_leaf(II_QueryIterator *child, double weight) {
    if (!is_node(child)) return false;
    NodeIter *n = NI(child);
    if (n->kind != NODE_RESULT || !n->rs || !n->rs->has_freqs || n->rs->n_children > (uint32_t)kIIMaxLists || n->host_ready) return false;
    II_ResultSet *inner = n->rs;
    n->rs = nullptr; // consumed either way
    II_PostingList *pl = II_ResultSet_IntoChild(inner, n->terms.data(), weight, 0);
    if (!pl) {
        n->kind = NODE_EMPTY;
        return false;
    }
    n->kind = NODE_LEAF;
    n->pl = pl;
    n->owns_pl = true;
    n->term = II_TermParams{weight, 1.0, 1.0};
    return true;
}

// NOT / OPTIONAL over one of OUR term leaves or nested AND / OR nodes (RS/rqe_iterators/src/not.rs, optional.rs): inside an AND
// they become an exclusion / an optional contribution of the membership kernel; read on their own they walk 1..max_doc_id.
II_QueryIterator *II_NewNotIterator(II_QueryIterator *child, t_docId max_doc_id, double weight) {
    if (child_is_empty(child)) { // NOT of nothing = every document: needs the universe, which only the host's wildcard iterator has
        if (child && child->Free) child->Free(child);
        return nullptr;
    }
    if (is_node(child) && NI(child)->kind == NODE_RESULT && !nested_node_to_leaf(child, 1.0)) return nullptr;
    if (!is_node(child) || NI(child)->kind != NODE_LEAF || NI(child)->mode != LEAF_REQUIRED) return nullptr;
    NodeIter *n = NI(child);
    n->mode = LEAF_NOT;
    n->max_doc_id = max_doc_id;
    n->base.type = 8; // IteratorType_Not
    n->cur.res.weight = weight;
    n->term.weight = 0.0; // a NOT child contributes a virtual result: nothing to the score (default.c:289-297)
    return child;
}
II_QueryIterator *II_NewOptionalIterator(II_QueryIterator *child, t_docId max_doc_id, double weight) {
    if (is_node(child) && NI(child)->kind == NODE_RESULT && !nested_node_to_leaf(child, weight)) return nullptr;
    if (!is_node(child) || NI(child)->kind != NODE_LEAF || NI(child)->mode != LEAF_REQUIRED) return nullptr;
    NodeIter *n = NI(child);
    n->mode = LEAF_OPTIONAL;
    n->max_doc_id = max_doc_id;
    n->base.type = 10; // IteratorType_Optional
    n->cur.res.weight = weight;
    n->term.weight = weight; // optional.rs:260: the weight is applied to real hits only; misses are virtual (score 0)
    return child;
}

static II_QueryIterator *build_aggregate(II_QueryIterator **its, size_t num, bool is_union, bool quick_exit, double weight,
                                         const PhraseSpec *phrase = nullptr) {
    auto free_children = [&] {
        for (size_t i = 0; i < num; i++)
            if (its[i] && its[i]->Free) its[i]->Free(its[i]);
        host_free(its);
    };
    // reduction rules (intersection.rs:363-417, union_reducer.rs:30-66)
    std::vector<II_QueryIterator *> kids;
    for (size_t i = 0; i < num; i++) {
        II_QueryIterator *c = its[i];
        const bool wildcard = c && (c->type == 12 /* Wildcard */ || c->type == 2 /* InvIdxWildcard */);
        if (!is_union) {
            if (child_is_empty(c)) { // any empty child -> the AND is empty
                free_children();
                return II_NewEmptyIterator();
            }
            if (wildcard) continue; // stripped (every document matches)
        } else if (child_is_empty(c)) {
            continue; // dropped
        }
        kids.push_back(c);
    }
    if (is_union && quick_exit) { // union_reducer.rs:41-53: a quick union with a wildcard child IS that wildcard
        for (size_t k = 0; k < kids.size(); k++)
            if (kids[k]->type == 12 /* Wildcard */ || kids[k]->type == 2 /* InvIdxWildcard */) {
                II_QueryIterator *keep = kids[k];
                for (size_t i = 0; i < num; i++)
                    if (its[i] && its[i] != keep && its[i]->Free) its[i]->Free(its[i]);
                host_free(its);
                return keep;
            }
    }
    if (kids.empty()) {
        // all wildcards -> the last one is returned (AND); nothing left -> empty (OR)
        II_QueryIterator *keep = nullptr;
        if (!is_union)
            for (size_t i = num; i-- > 0;)
                if (its[i]) {
                    keep = its[i];
                    break;
                }
        for (size_t i = 0; i < num; i++)
            if (its[i] && its[i] != keep && its[i]->Free) its[i]->Free(its[i]);
        host_free(its);
        return keep ? keep : II_NewEmptyIterator();
    }
    if (kids.size() == 1 && !(is_node(kids[0]) && NI(kids[0])->mode == LEAF_NOT)) { // one survivor -> the child itself
        II_QueryIterator *keep = kids[0];
        for (size_t i = 0; i < num; i++)
            if (its[i] && its[i] != keep && its[i]->Free) its[i]->Free(its[i]);
        host_free(its);
        return keep;
    }
    if (kids.size() > (size_t)(is_union ? kIIMaxUnionLists : kIIMaxLists)) {
        free_children();
        return nullptr;
    }
    std::vector<ChildView> views(kids.size());
    bool ok = true;
    for (size_t i = 0; i < kids.size() && ok; i++) ok = child_view(kids[i], views[i], phrase != nullptr);
    NodeIter *out = nullptr;
    if (ok) {
        std::vector<II_PostingList *> pls;
        std::vector<int> modes;
        std::vector<II_TermParams> terms;
        std::vector<std::string> strs;
        for (auto &v : views) {
            pls.push_back(v.pl);
            modes.push_back((int)v.mode);
            terms.push_back(v.term);
            strs.push_back(v.str);
        }
        bool any_mode = false, any_required = false;
        for (int m : modes) any_mode |= m != LEAF_REQUIRED, any_required |= m == LEAF_REQUIRED;
        II_ResultSet *rs = nullptr;
        if (is_union)
            rs = any_mode ? nullptr : II_Union(pls.data(), pls.size(), quick_exit ? 1 : 0);
        else if (phrase)
            rs = any_required ? II_IntersectPhrase(pls.data(), modes.data(), pls.size(),
                                                   phrase->max_slop == 0xFFFFFFFFu ? -1 : (int32_t)phrase->max_slop, phrase->in_order)
                              : nullptr;
        else if (!any_mode)
            rs = II_Intersect(pls.data(), pls.size());
        else if (any_required)
            rs = II_IntersectEx(pls.data(), modes.data(), pls.size());
        if (rs) {
            out = new_node(NODE_RESULT, is_union ? II_IteratorType_Union : II_IteratorType_Intersect, weight);
            out->rs = rs;
            out->terms = terms;
            out->term_strs = strs;
            out->agg_weight = weight;
        }
    }
    for (auto &v : views)
        if (v.temp) delete v.pl;
    free_children();
    return out ? &out->base : nullptr;
}

// RS/headers/iterators_ffi.h:309.  max_slop >= 0 / in_order (phrase constraints) are evaluated on the device when every child
// is one of OUR term leaves carrying its term positions (a codec with offsets, decoded with offsets kept) or a nested B200
// AND / OR (its children's positions are merged like the reference's aggregate offset iterator), at most kPhraseMaxLists
// children; for anything else (foreign children, leaves without positions) NULL is returned BEFORE anything is consumed and
// the caller keeps the reference's own iterator for that node.
II_QueryIterator *NewIntersectionIterator(II_QueryIterator **its, size_t num, int32_t max_slop, bool in_order, double weight) {
    if (!its || num == 0) {
        if (its) host_free(its);
        return II_NewEmptyIterator();
    }
    if (max_slop >= 0 || in_order) {
        if (num > (size_t)kPhraseMaxLists) return nullptr;
        for (size_t i = 0; i < num; i++) {
            II_QueryIterator *c = its[i];
            if (!c) return nullptr;
            if (child_is_empty(c)) continue; // reduces the AND to empty whatever the constraint
            if (!is_node(c)) return nullptr;
            if (NI(c)->kind == NODE_RESULT && NI(c)->rs) { // a nested AND / OR: the positions of its children are merged
                if (!NI(c)->rs->has_freqs || NI(c)->rs->n_children > (uint32_t)kIIMaxLists || NI(c)->host_ready) return nullptr;
                continue;
            }
            if (NI(c)->kind == NODE_WILDCARD) continue; // stripped from the AND
            if (NI(c)->kind != NODE_LEAF || !NI(c)->pl) return nullptr;
            if (NI(c)->mode != LEAF_NOT && !NI(c)->pl->d_off_len) return nullptr;
        }
        const PhraseSpec ph{max_slop < 0 ? 0xFFFFFFFFu : (uint32_t)max_slop, in_order};
        return build_aggregate(its, num, false, false, weight, &ph);
    }
    return build_aggregate(its, num, false, false, weight);
}
// RS/headers/iterators_ffi.h:594 (type_, q_str and config only steer the reference's flat / heap choice and its profile output)
II_QueryIterator *NewUnionIterator(II_QueryIterator **its, int32_t num, bool quick_exit, double weight, int type_, const char *q_str,
                                   const void *config) {
    (void)type_;
    (void)q_str;
    (void)config;
    if (!its || num <= 0) {
        if (its) host_free(its);
        return II_NewEmptyIterator();
    }
    return build_aggregate(its, (size_t)num, true, quick_exit, weight);
}

// ---- scorer extension ------------------------------------------------------------------------------
} // extern "C" (templates below)
namespace {
struct RSIndexStatsC { // src/redisearch.h:245-249
    size_t numDocs, numTerms;
    double avgDocLen;
};
struct ScoringFunctionArgsC { // src/redisearch.h:254-274
    void *extdata;
    const void *qdata;
    size_t qdatalen;
    RSIndexStatsC indexStats;
    void *scrExp;
    int (*GetSlop)(const void *res);
    uint64_t tanhFactor;
};
typedef double (*RSScoringFunctionC)(const ScoringFunctionArgsC *ctx, const void *res, const void *dmd, double minScore);
struct RSExtensionCtxC { // src/redisearch.h:282-287
    int (*RegisterScoringFunction)(const char *alias, RSScoringFunctionC func, void (*ff)(void *), void *privdata);
    int (*RegisterQueryExpander)(const char *alias, void *exp, void (*ff)(void *), void *privdata);
};

// ---- EXPLAINSCORE: the result tree of ONE hit read back from the device --------------------------------------------
// column i of a [n][stride] device array
bool fetch_column(const uint32_t *d, size_t stride, uint32_t n, size_t i, uint32_t *out) {
    return cudaMemcpy2D(out, 4, d + i, stride * 4, 4, n, cudaMemcpyDeviceToHost) == cudaSuccess;
}
// The reference's RSIndexResult tree for hit i of rs (document `doc`): children in aggregate order, a union's matching children only,
// NOT / absent OPTIONAL children of an intersection as virtual results, nested sets recursively through the hit's position in them.
bool hit_tree(const II_ResultSet *rs, const II_TermParams *terms, const std::vector<std::string> &strs, double weight, size_t i, uint32_t doc,
              iiexplain::TreeNode &out) {
    const uint32_t n = rs->n_children;
    if (n == 0 || n > (uint32_t)kIIMaxLists || !rs->has_freqs || i >= rs->len) return false;
    out = iiexplain::TreeNode();
    out.kind = rs->is_union ? iiexplain::Union : iiexplain::Intersection;
    out.weight = weight;
    uint32_t fr[kIIMaxLists], pos[kIIMaxLists];
    if (!fetch_column(rs->d_freqs, rs->cap, n, i, fr)) return false;
    const bool have_pos = rs->d_hit_pos != nullptr;
    if (have_pos && !fetch_column(rs->d_hit_pos, rs->cap, n, i, pos)) return false;
    // aggregate order: the constructor's for an intersection, the active array's epoch for a flat union (UnionOrder)
    uint32_t order[kIIMaxLists], cnt = n;
    for (uint32_t c = 0; c < n; c++) order[c] = c;
    if (rs->is_union && rs->h_order) {
        const UnionOrder &uo = *rs->h_order;
        uint32_t e = 0;
        while (e + 1 < uo.n_epochs && doc > uo.bound[e]) e++;
        cnt = uo.n_active[e];
        for (uint32_t c = 0; c < cnt; c++) order[c] = uo.perm[e][c];
    }
    for (uint32_t ci = 0; ci < cnt; ci++) {
        const uint32_t c = order[ci];
        const bool there = have_pos ? pos[c] != 0xFFFFFFFFu : fr[c] != 0;
        if (rs->is_union && !there) continue;
        iiexplain::TreeNode kid;
        const uint8_t tag = c < rs->child_tag.size() ? rs->child_tag[c] : 4;
        if (!there || tag == 8) { // NOT / absent OPTIONAL: a virtual result without weight; a wildcard child: virtual, freq 1
            kid.kind = iiexplain::Virtual;
            kid.freq = there ? fr[c] : 0;
            kid.weight = there ? terms[rs->child_order[c]].weight : 0.0;
        } else if (c < rs->nested.size() && rs->nested[c]) {
            const NestedSet *ns = rs->nested[c].get();
            if (!have_pos || !hit_tree(ns->rs.get(), ns->terms.data(), ns->term_strs, ns->weight, pos[c], doc, kid)) return false;
        } else {
            const II_TermParams &t = terms[rs->child_order[c]];
            kid.kind = tag == 16 || tag == 32 ? iiexplain::Numeric : iiexplain::Term;
            kid.freq = fr[c];
            kid.weight = t.weight;
            kid.idf = t.idf;
            kid.bm25_idf = t.bm25_idf;
            const uint32_t si = rs->child_order[c];
            if (si < strs.size()) kid.term = strs[si];
        }
        out.freq += kid.freq;
        out.kids.push_back(std::move(kid));
    }
    return true;
}
void *host_calloc(size_t n, size_t sz) {
    void *p = host_alloc(n * sz);
    if (p) memset(p, 0, n * sz);
    return p;
}
struct ScoreExplainC { // src/score_explain.h:20-24
    char *str;
    int numChildren;
    ScoreExplainC *children;
};
// the explanation into nodes owned by the host's allocator: `dst` is filled in place (str, a children array of its own)
bool explain_to_host(const iiexplain::Explain &e, ScoreExplainC *dst) {
    char *str = static_cast<char *>(host_alloc(e.str.size() + 1));
    if (!str) return false;
    memcpy(str, e.str.c_str(), e.str.size() + 1);
    if (dst->str) host_free(dst->str);
    dst->str = str;
    dst->numChildren = 0;
    dst->children = nullptr;
    if (e.kids.empty()) return true;
    dst->children = static_cast<ScoreExplainC *>(host_calloc(e.kids.size(), sizeof(ScoreExplainC)));
    if (!dst->children) return false;
    dst->numChildren = (int)e.kids.size();
    for (size_t k = 0; k < e.kids.size(); k++)
        if (!explain_to_host(e.kids[k], &dst->children[k])) return false;
    return true;
}

template <int kScorer>
double b200_scorer(const ScoringFunctionArgsC *args, const void *res_v, const void *dmd, double min_score) {
    (void)dmd;
    const II_IndexResult *res = static_cast<const II_IndexResult *>(res_v);
    uint64_t magic = 0;
    NodeIter *it = nullptr;
    if (res && res->data.tag == II_ResultData_Metric) {
        memcpy(&magic, res->data._rest, 8);
        memcpy(&it, res->data._rest + 8, 8);
    }
    if (magic != kNodeMagic || !it || it->magic != kNodeMagic) {
        static bool warned = false;
        if (!warned) fprintf(stderr, "ii_b200: a *.B200 scorer was called on a result that does not come from a B200 iterator; returning 0\n");
        warned = true;
        return 0.0;
    }
    if (it->scored_with != kScorer) { // first call for this result set: score every hit on the device, once
        if (!node_materialise(it) || !it->rs || !node_host(it)) return 0.0;
        II_IndexStats st{args->indexStats.numDocs, args->indexStats.numTerms, args->indexStats.avgDocLen};
        // terms are stored in the order of the constructor's `its`, which is what II_Score expects
        if (kScorer == II_SCORER_HAMMING) {
            if (II_ScoreHamming(it->rs, it->docs, args->qdata, args->qdatalen) != 0) return 0.0;
        } else if (II_Score(it->rs, (II_Scorer)kScorer, it->terms.data(), it->agg_weight, &st, it->docs, min_score,
                            args->tanhFactor ? args->tanhFactor : 4) != 0)
            return 0.0;
        if (II_ResultSet_Fetch(it->rs, nullptr, it->cur.scores.data(), nullptr) != 0) return 0.0;
        it->scored_with = kScorer;
    }
    // `res` is the iterator's current result: pos points one past it
    const size_t i = it->cur.pos ? it->cur.pos - 1 : 0;
    const double score = i < it->cur.scores.size() ? it->cur.scores[i] : 0.0;
    if (args->scrExp) {
        // EXPLAINSCORE (src/result_processor.c:582-584 hands the node to the reply, src/score_explain.c:19-21 prints `str`
        // unconditionally): the hit's result tree is read back from the device and explained with the reference's own strings
        // (ii_explain.cpp); the node RPScorer handed in becomes the root, filled in place
        auto *e = static_cast<ScoreExplainC *>(args->scrExp);
        iiexplain::Explain ex;
        bool itemised = false;
        if (kScorer == II_SCORER_HAMMING) {
            iiexplain::explain_hamming(score, args->qdatalen, ex);
            itemised = true;
        } else if (i < it->cur.ids.size()) {
            Ctx &c = ctx();
            std::lock_guard<std::mutex> g(c.mu);
            const uint32_t doc = (uint32_t)it->cur.ids[i];
            iiexplain::TreeNode tree;
            iiexplain::DocParams dp;
            dp.avg_doc_len = args->indexStats.avgDocLen;
            dp.doc_score = 1.0f;
            dp.max_freq = 1;
            bool ok = c.init() && cudaStreamSynchronize(c.stream) == cudaSuccess && hit_tree(it->rs, it->terms.data(), it->term_strs, it->agg_weight, i, doc, tree);
            const II_DocTable *dt = it->docs;
            if (ok && dt && doc <= dt->max_doc) {
                if (dt->d_len) ok = ok && cudaMemcpy(&dp.doc_len, dt->d_len + doc, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
                if (dt->d_score) ok = ok && cudaMemcpy(&dp.doc_score, dt->d_score + doc, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
                if (dt->d_maxf) ok = ok && cudaMemcpy(&dp.max_freq, dt->d_maxf + doc, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
            }
            uint32_t slop = 1;
            if (ok && (kScorer == II_SCORER_BM25 || kScorer == II_SCORER_TFIDF || kScorer == II_SCORER_TFIDF_DOCNORM)) {
                if (it->rs->d_slop)
                    ok = cudaMemcpy(&slop, it->rs->d_slop + i, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
                else
                    slop = tree.kids.size() <= 1 ? 1u : (uint32_t)tree.kids.size() - 1u; // IndexResult_MinOffsetDelta without offsets
            }
            if (ok) {
                if (it->kind == NODE_LEAF && tree.kids.size() == 1) { // a term read directly: the reference's root IS the term result
                    iiexplain::TreeNode only = std::move(tree.kids[0]);
                    tree = std::move(only);
                }
                iiexplain::explain_score(kScorer, tree, dp, (int)slop, min_score, args->tanhFactor ? args->tanhFactor : 4, ex);
                itemised = true;
            }
        }
        if (!itemised) {
            static const char *const kNames[] = {"BM25STD", "BM25", "TFIDF", "TFIDF.DOCNORM", "DOCSCORE", "BM25STD.TANH", "DISMAX", "HAMMING"};
            char buf[160];
            snprintf(buf, sizeof(buf), "Final %s.B200 : %.2f (per-term break-down not available for this result)", kNames[kScorer], score);
            ex = iiexplain::Explain();
            ex.str = buf;
        }
        explain_to_host(ex, e);
    }
    return score;
}
} // namespace
extern "C" {

// Loaded by Extension_LoadDynamic (dlopen + dlsym "RS_ExtensionInit", src/extension.c:121-145).  Registers the device
// counterparts of the default scorers under <NAME>.B200; FT.SEARCH ... SCORER BM25STD.B200 then returns, per result, the
// score computed on the device for the whole result set.  0 = REDISEARCH_OK.
int RS_ExtensionInit(void *ctx_v) {
    auto *ctx = static_cast<RSExtensionCtxC *>(ctx_v);
    if (!ctx || !ctx->RegisterScoringFunction) return 1;
    int rc = 0;
    rc |= ctx->RegisterScoringFunction("BM25STD.B200", b200_scorer<II_SCORER_BM25STD>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("BM25.B200", b200_scorer<II_SCORER_BM25>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("TFIDF.B200", b200_scorer<II_SCORER_TFIDF>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("TFIDF.DOCNORM.B200", b200_scorer<II_SCORER_TFIDF_DOCNORM>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("DOCSCORE.B200", b200_scorer<II_SCORER_DOCSCORE>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("BM25STD.TANH.B200", b200_scorer<II_SCORER_BM25STD_TANH>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("DISMAX.B200", b200_scorer<II_SCORER_DISMAX>, nullptr, nullptr);
    rc |= ctx->RegisterScoringFunction("HAMMING.B200", b200_scorer<II_SCORER_HAMMING>, nullptr, nullptr);
    return rc ? 1 : 0;
}

II_Stats II_GetStats(bool reset) {
    Ctx &c = ctx();
    std::lock_guard<std::mutex> g(c.mu);
    II_Stats s = c.stats;
    if (reset) c.stats = II_Stats{};
    return s;
}
// Coordinator-side merge of per-shard top-N lists (postings sharded by docId range, SURVEY.md §8e): the shards'
// lists are disjoint in docId, so the global top-N by cmpByScore (score desc, docId asc —
// src/result_processor.c:834-850) is the top-N of their union.  Host code, no device needed.
size_t II_MergeShardTopN(const double *scores, const uint64_t *doc_ids, const size_t *counts, size_t num_shards, size_t per_shard,
                         size_t n, uint64_t *out_ids, double *out_scores) {
    std::vector<std::pair<double, uint64_t>> all;
    for (size_t g = 0; g < num_shards; g++)
        for (size_t i = 0; i < std::min(counts[g], per_shard); i++) all.emplace_back(scores[g * per_shard + i], doc_ids[g * per_shard + i]);
    const size_t k = std::min(n, all.size());
    std::partial_sort(all.begin(), all.begin() + k, all.end(), [](const std::pair<double, uint64_t> &a, const std::pair<double, uint64_t> &b) {
        return a.first > b.first || (a.first == b.first && a.second < b.second);
    });
    for (size_t i = 0; i < k; i++) {
        out_scores[i] = all[i].first;
        out_ids[i] = all[i].second;
    }
    return k;
}
const char *II_Version(void) { return "ii_b200 0.1 (sm_90a)"; }

// EXPLAINSCORE of one result given as a flattened tree (node 0 the root, parent[i] < i, children in index order; kind 0 term,
// 1 intersection, 2 union, 3 virtual, 4 numeric; term_str: every term leaf's text, may be NULL): the explanation the reference's
// scorer builds (src/ext/default.c), serialised one node per line as "<depth> <string>\n" in pre-order.  Host code (no device):
// what the *.B200 scorers call when ScoringFunctionArgs.scrExp is set.  Returns the bytes needed (excluding the NUL).
size_t II_ExplainTree(int scorer, size_t n_nodes, const int32_t *parent, const int32_t *kind, const uint32_t *freq, const double *weight,
                      const double *idf, const double *bm25_idf, const char *term_str, uint32_t doc_len, uint32_t max_freq, float doc_score,
                      double avg_doc_len, int slop, double min_score, uint64_t tanh_factor, double *score_out, char *buf, size_t cap) {
    if (!n_nodes) return 0;
    std::vector<iiexplain::TreeNode> flat(n_nodes);
    for (size_t i = 0; i < n_nodes; i++) {
        flat[i].kind = kind[i];
        flat[i].freq = freq[i];
        flat[i].weight = weight[i];
        flat[i].idf = idf[i];
        flat[i].bm25_idf = bm25_idf[i];
        if (term_str) flat[i].term = term_str;
    }
    for (size_t i = n_nodes; i-- > 1;) { // children were appended after their parents: fold from the back, keeping index order
        if (parent[i] < 0 || (size_t)parent[i] >= i) return 0;
        iiexplain::TreeNode &p = flat[parent[i]];
        p.kids.insert(p.kids.begin(), std::move(flat[i]));
    }
    iiexplain::Explain e;
    const iiexplain::DocParams d{doc_len, max_freq, doc_score, avg_doc_len};
    const double score = iiexplain::explain_score(scorer, flat[0], d, slop, min_score, tanh_factor, e);
    if (score_out) *score_out = score;
    std::string out;
    std::function<void(const iiexplain::Explain &, int)> walk = [&](const iiexplain::Explain &n, int depth) {
        out += std::to_string(depth) + " " + n.str + "\n";
        for (const auto &k : n.kids) walk(k, depth + 1);
    };
    walk(e, 0);
    if (buf && cap) {
        const size_t m = std::min(cap - 1, out.size());
        memcpy(buf, out.data(), m);
        buf[m] = 0;
    }
    return out.size();
}

} // extern "C"
