// The one exchange step of the sharded KNN query, behind the C-ABI: every rank scans its row shard, ONE ncclAllGather
// moves the per-shard top-k (labels + scores in one packed block per rank) over NVLink, every rank merges on device
// by (score, label) — the coordinator's knnPostProcess (src/module.c:3139-3176) with the comparator of
// VS/utils/query_result_utils.h:19-23.  NCCL is bound at run time (dlopen of libnccl.so.2: the copy the host process
// already loaded — PyTorch's, or the system library for a C host), so libvecsim_b200.so has no link-time dependency
// on it and single-GPU users never load it.
#include "topk_common.cuh"
#include "vecsim_index.h"

#include <dlfcn.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <mutex>

namespace {
using rsb200::FlatIndex;

typedef int ncclResult_t;
typedef void *ncclComm_t;
struct Id128 { // ncclUniqueId
    char internal[128];
};
struct NcclApi {
    ncclResult_t (*GetUniqueId)(void *id128) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *comm, int nranks, Id128 id /* by value, as in nccl.h */, int rank) = nullptr;
    ncclResult_t (*AllGather)(const void *send, void *recv, size_t count, int dtype, ncclComm_t comm, cudaStream_t s) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t comm) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
NcclApi &nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *override_path = getenv("VECSIM_B200_NCCL_LIB");
        const char *names[] = {override_path, "libnccl.so.2", "libnccl.so"};
        void *h = nullptr;
        for (const char *n : names) {
            if (!n || !*n) continue;
            h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (h) break;
        }
        if (!h) {
            fprintf(stderr, "[vecsim_b200] cannot load NCCL (libnccl.so.2): %s\n", dlerror());
            return;
        }
        api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
        api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
        api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(h, "ncclAllGather"));
        api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
        api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
        api.ok = api.GetUniqueId && api.CommInitRank && api.AllGather && api.CommDestroy;
    });
    return api;
}

bool nccl_ok(ncclResult_t r, const char *what) {
    if (r == 0) return true;
    const char *msg = nccl().GetErrorString ? nccl().GetErrorString(r) : "?";
    fprintf(stderr, "[vecsim_b200] NCCL error in %s: %s\n", what, msg);
    return false;
}
inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }
} // namespace

struct VecSimB200_ShardGroup {
    int rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    cudaStream_t stream = nullptr; // host-facing entry point
    // packed exchange block of one rank: [labels int64 x nq*k][scores float x nq*k], padded to 16 bytes
    uint8_t *d_send = nullptr, *d_recv = nullptr;
    size_t block_cap = 0;
    // host-facing entry point: staged queries and merged results
    uint8_t *d_q = nullptr, *h_q = nullptr;
    size_t q_cap = 0;
    int64_t *d_labels = nullptr, *h_labels = nullptr;
    float *d_scores = nullptr, *h_scores = nullptr;
    size_t out_cap = 0;
    std::mutex mu;

    bool need_block(size_t bytes) {
        if (bytes <= block_cap) return true;
        cudaFree(d_send);
        cudaFree(d_recv);
        d_send = d_recv = nullptr;
        block_cap = 0;
        if (cudaMalloc(&d_send, bytes) != cudaSuccess || cudaMalloc(&d_recv, bytes * (size_t)world) != cudaSuccess) return false;
        block_cap = bytes;
        return true;
    }
    bool need_host_io(size_t qbytes, size_t nout) {
        if (qbytes > q_cap) {
            cudaFree(d_q);
            cudaFreeHost(h_q);
            d_q = h_q = nullptr;
            q_cap = 0;
            if (cudaMalloc(&d_q, qbytes) != cudaSuccess || cudaMallocHost(&h_q, qbytes) != cudaSuccess) return false;
            q_cap = qbytes;
        }
        if (nout > out_cap) {
            cudaFree(d_labels);
            cudaFree(d_scores);
            cudaFreeHost(h_labels);
            cudaFreeHost(h_scores);
            d_labels = h_labels = nullptr;
            d_scores = h_scores = nullptr;
            out_cap = 0;
            if (cudaMalloc(&d_labels, nout * 8) != cudaSuccess || cudaMalloc(&d_scores, nout * 4) != cudaSuccess ||
                cudaMallocHost(&h_labels, nout * 8) != cudaSuccess || cudaMallocHost(&h_scores, nout * 4) != cudaSuccess)
                return false;
            out_cap = nout;
        }
        return true;
    }
};

namespace {
// Counted exchange block of one rank (DESIGN.md §6.1): [labels int64 x nq*w][scores float x nq*w][counts u32 x nq], padded to 16 bytes
size_t list_block_bytes(size_t nq, size_t w) { return align16(nq * w * 12 + nq * 4); }

// Refusals every rank makes alike, from the arguments they share, before anything is enqueued
bool shared_mode_ok(const VecSimQueryParams *qp) {
    const int m = qp ? (int)qp->searchMode : (int)EMPTY_MODE;
    return m == EMPTY_MODE || m == HYBRID_ADHOC_BF || m == HYBRID_BATCHES;
}
bool shared_range_ok(size_t nq, size_t cap, VecSimQueryReply_Order order) {
    return cap >= 1 && cap <= rsb200::kRangeDeviceMaxCap && (order == BY_SCORE || order == BY_ID) && nq <= (1ull << 31);
}

// The body of the list collectives: `local(labels, scores, counts)` is this rank's local call, writing its rows straight into the
// send block; ONE all-gather; the list merge.  A local refusal (its shard, its filters, a failed flush) still takes part in the
// exchange with a failed block (counts UINT32_MAX), so no rank is left waiting in the all-gather and every rank's merged rows come
// out failed; the call then returns the local code.
template <class Local>
int list_collective(VecSimB200_ShardGroup *g, size_t nq, size_t w, bool range, VecSimQueryReply_Order order, int64_t *d_out_labels,
                    float *d_out_scores, uint32_t *d_out_counts, cudaStream_t st, Local local) {
    const size_t n = nq * w, block = list_block_bytes(nq, w);
    {
        std::lock_guard<std::mutex> lk(g->mu);
        if (!g->need_block(block)) return -1;
    }
    const int rc = local(reinterpret_cast<int64_t *>(g->d_send), reinterpret_cast<float *>(g->d_send + n * 8),
                         reinterpret_cast<uint32_t *>(g->d_send + n * 12));
    if (rc != 0 && cudaMemsetAsync(g->d_send, 0xFF, block, st) != cudaSuccess) return -1;
    if (!nccl_ok(nccl().AllGather(g->d_send, g->d_recv, block, /* ncclInt8 */ 0, g->comm, st), "ncclAllGather")) return -1;
    if (rsb200::launch_merge_lists(g->d_recv, block, (uint32_t)g->world, (uint32_t)nq, (uint32_t)w, range, order == BY_ID, d_out_labels,
                                   d_out_scores, d_out_counts, st, nullptr) != cudaSuccess)
        return -1;
    return rc;
}
} // namespace

extern "C" {

size_t VecSimB200_ShardListBlockBytes(size_t nq, size_t w) { return list_block_bytes(nq, w); }

int VecSimB200_MergeShardListBlocks(const void *d_blocks, size_t G, size_t nq, size_t w, int range, VecSimQueryReply_Order order,
                                    int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts, void *stream) {
    if (G == 0 || G > 0xFFFFFFFFull || w == 0 || w > rsb200::kMaxListWidth || nq > (1ull << 31) || (range != 0 && range != 1) ||
        (order != BY_SCORE && order != BY_ID) || (order == BY_ID && range == 0))
        return -1;
    return rsb200::launch_merge_lists(d_blocks, list_block_bytes(nq, w), (uint32_t)G, (uint32_t)nq, (uint32_t)w, range == 1, order == BY_ID,
                                      d_out_labels, d_out_scores, d_out_counts, static_cast<cudaStream_t>(stream), nullptr) == cudaSuccess
               ? 0
               : -1;
}

int VecSimB200_ShardGroup_HybridTopKBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq, size_t k,
                                                const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                                VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                                uint32_t *d_out_counts, int *out_modes, void *stream) {
    if (!g || !shard) return -1;
    FlatIndex *ix = reinterpret_cast<FlatIndex *>(shard);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    if (g->world == 1)
        return ix->hybrid_topk_batch_device(d_queries, nq, k, d_doc_ids, d_counts, caps, queryParams, d_out_labels, d_out_scores, d_out_counts,
                                            out_modes, st);
    if (!shared_mode_ok(queryParams) || k > (size_t)rsb200::kMaxWideK || nq > (1ull << 31)) return -1;
    if (nq == 0 || k == 0) return 0;
    return list_collective(g, nq, k, false, BY_SCORE, d_out_labels, d_out_scores, d_out_counts, st, [&](int64_t *l, float *s, uint32_t *c) {
        return ix->hybrid_topk_batch_device(d_queries, nq, k, d_doc_ids, d_counts, caps, queryParams, l, s, c, out_modes, st);
    });
}

int VecSimB200_ShardGroup_RangeQueryBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq,
                                                const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_out_labels,
                                                float *d_out_scores, uint32_t *d_out_counts, void *stream) {
    if (!g || !shard) return -1;
    FlatIndex *ix = reinterpret_cast<FlatIndex *>(shard);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    if (g->world == 1) return ix->label_range_batch_device(d_queries, nq, d_radii, cap, order, d_out_labels, d_out_scores, d_out_counts, st);
    if (!shared_range_ok(nq, cap, order)) return -1;
    if (nq == 0) return 0;
    return list_collective(g, nq, cap, true, order, d_out_labels, d_out_scores, d_out_counts, st, [&](int64_t *l, float *s, uint32_t *c) {
        return ix->label_range_batch_device(d_queries, nq, d_radii, cap, order, l, s, c, st);
    });
}

int VecSimB200_ShardGroup_HybridRangeQueryBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq,
                                                      const float *d_radii, size_t cap, VecSimQueryReply_Order order,
                                                      const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                                      VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                                      uint32_t *d_out_counts, int *out_modes, void *stream) {
    if (!g || !shard) return -1;
    FlatIndex *ix = reinterpret_cast<FlatIndex *>(shard);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    if (g->world == 1)
        return ix->hybrid_range_batch_device(d_queries, nq, d_radii, cap, order, d_doc_ids, d_counts, caps, queryParams, d_out_labels,
                                             d_out_scores, d_out_counts, out_modes, st);
    if (!shared_mode_ok(queryParams) || !shared_range_ok(nq, cap, order)) return -1;
    if (nq == 0) return 0;
    return list_collective(g, nq, cap, true, order, d_out_labels, d_out_scores, d_out_counts, st, [&](int64_t *l, float *s, uint32_t *c) {
        return ix->hybrid_range_batch_device(d_queries, nq, d_radii, cap, order, d_doc_ids, d_counts, caps, queryParams, l, s, c, out_modes, st);
    });
}

// Exchange format of one shard: [labels int64 x nq*k][scores float x nq*k], padded to 16 bytes.
size_t VecSimB200_ShardBlockBytes(size_t nq, size_t k) { return align16(nq * k * 12); }

// G packed blocks (rank-major, as an all-gather of the blocks leaves them) -> merged [nq][k] by (score, label).  For hosts
// that move the blocks with their own transport instead of VecSimB200_ShardGroup.
int VecSimB200_MergeShardBlocks(const void *d_blocks, size_t G, size_t nq, size_t k, float *d_out_scores, int64_t *d_out_labels,
                                void *stream) {
    const size_t block = align16(nq * k * 12);
    const uint8_t *base = static_cast<const uint8_t *>(d_blocks);
    return rsb200::launch_merge_shards(reinterpret_cast<const float *>(base + nq * k * 8), reinterpret_cast<const int64_t *>(base),
                                       (uint32_t)G, (uint32_t)nq, (uint32_t)k, d_out_scores, d_out_labels,
                                       static_cast<cudaStream_t>(stream), nullptr, block / 4, block / 8) == cudaSuccess
               ? 0
               : -1;
}

int VecSimB200_ShardGroup_UniqueId(void *out128) {
    if (!nccl().ok || !out128) return -1;
    return nccl_ok(nccl().GetUniqueId(out128), "ncclGetUniqueId") ? 0 : -1;
}

VecSimB200_ShardGroup *VecSimB200_ShardGroup_New(const void *id128, int rank, int world) {
    if (world < 1 || rank < 0 || rank >= world) return nullptr;
    auto *g = new VecSimB200_ShardGroup();
    g->rank = rank;
    g->world = world;
    if (cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete g;
        return nullptr;
    }
    if (world > 1) {
        Id128 id;
        if (!nccl().ok || !id128) {
            cudaStreamDestroy(g->stream);
            delete g;
            return nullptr;
        }
        memcpy(&id, id128, sizeof(id));
        if (!nccl_ok(nccl().CommInitRank(&g->comm, world, id, rank), "ncclCommInitRank")) {
            cudaStreamDestroy(g->stream);
            delete g;
            return nullptr;
        }
    }
    return g;
}

void VecSimB200_ShardGroup_Free(VecSimB200_ShardGroup *g) {
    if (!g) return;
    if (g->stream) cudaStreamSynchronize(g->stream);
    if (g->comm) nccl().CommDestroy(g->comm);
    cudaFree(g->d_send);
    cudaFree(g->d_recv);
    cudaFree(g->d_q);
    cudaFreeHost(g->h_q);
    cudaFree(g->d_labels);
    cudaFree(g->d_scores);
    cudaFreeHost(g->h_labels);
    cudaFreeHost(g->h_scores);
    if (g->stream) cudaStreamDestroy(g->stream);
    delete g;
}

int VecSimB200_ShardGroup_Rank(const VecSimB200_ShardGroup *g) { return g ? g->rank : -1; }
int VecSimB200_ShardGroup_Size(const VecSimB200_ShardGroup *g) { return g ? g->world : 0; }

// Enqueued on `stream` (NULL = the legacy default stream), nothing is synchronised: local scan of this rank's shard
// -> one all-gather of the packed per-shard top-k -> G-way merge.  Every rank ends up with the merged [nq][k] answer.
int VecSimB200_ShardGroup_TopKBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *index, const void *d_queries, size_t nq, size_t k,
                                          int64_t *d_out_labels, float *d_out_scores, void *stream) {
    if (!g || !index) return -1;
    if (nq == 0 || k == 0) return 0;
    FlatIndex *ix = reinterpret_cast<FlatIndex *>(index);
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : cudaStreamLegacy;
    if (g->world == 1) return ix->topk_batch_device(d_queries, nq, k, d_out_labels, d_out_scores, st);
    const size_t n = nq * k, block = align16(n * 12);
    {
        std::lock_guard<std::mutex> lk(g->mu);
        if (!g->need_block(block)) return -1;
    }
    int64_t *send_labels = reinterpret_cast<int64_t *>(g->d_send);
    float *send_scores = reinterpret_cast<float *>(g->d_send + n * 8);
    if (ix->size() == 0) { // an empty shard still takes part in the exchange
        if (cudaMemsetAsync(g->d_send, 0xFF, block, st) != cudaSuccess) return -1;
    } else if (ix->topk_batch_device(d_queries, nq, k, send_labels, send_scores, st) != 0) {
        return -1;
    }
    if (!nccl_ok(nccl().AllGather(g->d_send, g->d_recv, block, /* ncclInt8 */ 0, g->comm, st), "ncclAllGather")) return -1;
    const float *rs = reinterpret_cast<const float *>(g->d_recv + n * 8);
    const int64_t *rl = reinterpret_cast<const int64_t *>(g->d_recv);
    return rsb200::launch_merge_shards(rs, rl, (uint32_t)g->world, (uint32_t)nq, (uint32_t)k, d_out_scores, d_out_labels, st, nullptr,
                                       block / 4, block / 8) == cudaSuccess
               ? 0
               : -1;
}

// The same end to end with HOST buffers: query blobs in (raw, as for VecSimIndex_TopKQuery), merged labels / distances
// out; H2D, the shard scan, the exchange, the merge and D2H all inside the call.  Collective: every rank calls it with
// the same queries.  Empty slots: label SIZE_MAX, score NaN.
int VecSimB200_ShardGroup_TopKBatch(VecSimB200_ShardGroup *g, VecSimIndex *index, const void *queryBlobs, size_t qstride, size_t nq, size_t k,
                                    size_t *out_labels, double *out_scores) {
    if (!g || !index) return -1;
    if (nq == 0 || k == 0) return 0;
    FlatIndex *ix = reinterpret_cast<FlatIndex *>(index);
    const size_t qpitch = align16(ix->query_blob_bytes());
    std::unique_lock<std::mutex> lk(g->mu);
    if (!g->need_host_io(qpitch * nq, nq * k)) return -1;
    lk.unlock();
    memset(g->h_q, 0, qpitch * nq);
    for (size_t i = 0; i < nq; i++) ix->preprocess_query(static_cast<const uint8_t *>(queryBlobs) + i * qstride, g->h_q + i * qpitch);
    if (cudaMemcpyAsync(g->d_q, g->h_q, qpitch * nq, cudaMemcpyHostToDevice, g->stream) != cudaSuccess) return -1;
    if (VecSimB200_ShardGroup_TopKBatchDevice(g, index, g->d_q, nq, k, g->d_labels, g->d_scores, g->stream) != 0) return -1;
    if (cudaMemcpyAsync(g->h_labels, g->d_labels, nq * k * 8, cudaMemcpyDeviceToHost, g->stream) != cudaSuccess ||
        cudaMemcpyAsync(g->h_scores, g->d_scores, nq * k * 4, cudaMemcpyDeviceToHost, g->stream) != cudaSuccess ||
        cudaStreamSynchronize(g->stream) != cudaSuccess)
        return -1;
    for (size_t i = 0; i < nq * k; i++) {
        out_labels[i] = g->h_labels[i] < 0 ? SIZE_MAX : (size_t)g->h_labels[i];
        out_scores[i] = g->h_labels[i] < 0 ? std::numeric_limits<double>::quiet_NaN() : (double)g->h_scores[i];
    }
    return 0;
}

} // extern "C"
