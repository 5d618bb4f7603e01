// extern "C" surface of libvecsim_b200.so — see include/vecsim_b200.h for the contract and the
// reference declaration each entry point replaces (VS/vec_sim.h, VS/query_results.h,
// VS/vec_sim.cpp:213-432, VS/query_results.cpp:23-93).
#include "vecsim_index.h"
#include "host_numeric.h"

#include <cerrno>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <strings.h>

using rsb200::AdhocCtx;
using rsb200::BatchIter;
using rsb200::FlatIndex;

struct VecSimBatchIterator : BatchIter {};
struct VecSimAdhocBfCtx : AdhocCtx {};

static inline FlatIndex *IX(VecSimIndex *i) { return reinterpret_cast<FlatIndex *>(i); }

extern "C" {

// ---------------------------------------------------------------------------------- lifetime
VecSimIndex *VecSimIndex_New(const VecSimParams *params) {
    if (!params || params->algo != VecSimAlgo_BF) return nullptr;
    return reinterpret_cast<VecSimIndex *>(FlatIndex::create(params->algoParams.bfParams, params->logCtx));
}

static size_t stored_size(VecSimType type, size_t dim, VecSimMetric metric) {
    size_t es = 0;
    switch (type) {
    case VecSimType_FLOAT32: es = 4; break;
    case VecSimType_FLOAT64: es = 8; break;
    case VecSimType_BFLOAT16:
    case VecSimType_FLOAT16: es = 2; break;
    case VecSimType_INT8:
    case VecSimType_UINT8: es = 1; break;
    case VecSimType_INT32: es = 4; break;
    case VecSimType_INT64: es = 8; break;
    }
    size_t s = es * dim;
    if (metric == VecSimMetric_Cosine && (type == VecSimType_INT8 || type == VecSimType_UINT8)) s += sizeof(float);
    return s;
}

size_t VecSimIndex_EstimateInitialSize(const VecSimParams *params) {
    if (!params || params->algo != VecSimAlgo_BF) return 0;
    // An empty index owns its host object, the pinned staging ring and no HBM yet.
    const BFParams &p = params->algoParams.bfParams;
    const size_t pitch = (stored_size(p.type, p.dim, p.metric) + 15) & ~(size_t)15;
    return sizeof(FlatIndex) + std::min<size_t>(32u << 20, pitch << 20);
}

size_t VecSimIndex_EstimateElementSize(const VecSimParams *params) {
    if (!params || params->algo != VecSimAlgo_BF) return 0;
    // brute_force_factory.cpp:129-134: vector + idToLabel entry + label map entry
    const BFParams &p = params->algoParams.bfParams;
    return stored_size(p.type, p.dim, p.metric) + sizeof(labelType) + sizeof(void *);
}

void VecSimIndex_Free(VecSimIndex *index) { delete IX(index); }

int VecSimIndex_AddVector(VecSimIndex *index, const void *blob, size_t label) { return IX(index)->add(blob, label); }
int VecSimIndex_DeleteVector(VecSimIndex *index, size_t label) { return IX(index)->remove(label); }
size_t VecSimIndex_IndexSize(VecSimIndex *index) { return IX(index)->size(); }

// ---------------------------------------------------------------------------------- queries
VecSimQueryReply *VecSimIndex_TopKQuery(VecSimIndex *index, const void *queryBlob, size_t k,
                                        VecSimQueryParams *queryParams, VecSimQueryReply_Order order) {
    if (rsb200::FlatIndex::microbatch_window_us() > 0) return IX(index)->topk_combined(queryBlob, k, queryParams, order);
    return IX(index)->topk(queryBlob, k, queryParams, order);
}

VecSimQueryReply *VecSimIndex_RangeQuery(VecSimIndex *index, const void *queryBlob, double radius,
                                         VecSimQueryParams *queryParams, VecSimQueryReply_Order order) {
    if (order != BY_ID && order != BY_SCORE) {
        IX(index)->log("warning", "Possible order values are only 'BY_ID' or 'BY_SCORE'");
        return nullptr;
    }
    if (radius < 0) {
        IX(index)->log("warning", "radius must be non-negative");
        return nullptr;
    }
    return IX(index)->range(queryBlob, radius, queryParams, order);
}

double VecSimIndex_GetDistanceFrom_Unsafe(VecSimIndex *index, size_t label, const void *blob) {
    return IX(index)->distance_from(label, blob);
}

bool VecSimIndex_PreferAdHocSearch(VecSimIndex *index, size_t subsetSize, size_t k, bool initial_check) {
    return IX(index)->prefer_adhoc(subsetSize, k, initial_check);
}

// vec_sim.cpp:127-211, 270-343 restricted to what a FLAT index accepts: every HNSW/SVS-only
// parameter is UnknownParam for VecSimAlgo_BF exactly as upstream.
static bool parse_positive_ll(const VecSimRawParam &p, long long *out) {
    // utils/vec_utils.cpp validate_positive_integer_param: whole string must parse, value > 0
    if (!p.value || p.valLen == 0) return false;
    char *end = nullptr;
    errno = 0;
    long long v = strtoll(p.value, &end, 10);
    if (errno != 0 || end != p.value + p.valLen || v <= 0) return false;
    *out = v;
    return true;
}

VecSimResolveCode VecSimIndex_ResolveParams(VecSimIndex *index, VecSimRawParam *rparams, int paramNum,
                                            VecSimQueryParams *qparams, VecsimQueryType query_type) {
    if (!qparams || (!rparams && paramNum != 0)) return VecSimParamResolverErr_NullParam;
    memset(qparams, 0, sizeof(*qparams));
    for (int i = 0; i < paramNum; i++) {
        const VecSimRawParam &rp = rparams[i];
        if (!strcasecmp(rp.name, "BATCH_SIZE")) {
            long long v;
            if (query_type != QUERY_TYPE_HYBRID) return VecSimParamResolverErr_InvalidPolicy_NHybrid;
            if (qparams->batchSize != 0) return VecSimParamResolverErr_AlreadySet;
            if (!parse_positive_ll(rp, &v)) return VecSimParamResolverErr_BadValue;
            qparams->batchSize = (size_t)v;
        } else if (!strcasecmp(rp.name, "HYBRID_POLICY")) {
            if (query_type != QUERY_TYPE_HYBRID) return VecSimParamResolverErr_InvalidPolicy_NHybrid;
            if (qparams->searchMode != 0) return VecSimParamResolverErr_AlreadySet;
            if (!strcasecmp(rp.value, VECSIM_POLICY_BATCHES))
                qparams->searchMode = HYBRID_BATCHES;
            else if (!strcasecmp(rp.value, VECSIM_POLICY_ADHOC_BF))
                qparams->searchMode = HYBRID_ADHOC_BF;
            else
                return VecSimParamResolverErr_InvalidPolicy_NExits;
        } else if (!strcasecmp(rp.name, "EPSILON")) {
            return VecSimParamResolverErr_UnknownParam; // HNSW / SVS only
        } else if (!strcasecmp(rp.name, "EF_RUNTIME") || !strcasecmp(rp.name, "RERANK") ||
                   !strcasecmp(rp.name, "SEARCH_WINDOW_SIZE") || !strcasecmp(rp.name, "SEARCH_BUFFER_CAPACITY") ||
                   !strcasecmp(rp.name, "USE_SEARCH_HISTORY")) {
            return VecSimParamResolverErr_UnknownParam;
        } else {
            return VecSimParamResolverErr_UnknownParam;
        }
    }
    if (qparams->searchMode == HYBRID_ADHOC_BF && qparams->batchSize > 0)
        return VecSimParamResolverErr_InvalidPolicy_AdHoc_With_BatchSize;
    if (qparams->searchMode != 0) IX(index)->set_last_mode(qparams->searchMode);
    return VecSimParamResolver_OK;
}

// ---------------------------------------------------------------------------------- batch iterator
VecSimBatchIterator *VecSimBatchIterator_New(VecSimIndex *index, const void *queryBlob, VecSimQueryParams *queryParams) {
    return static_cast<VecSimBatchIterator *>(IX(index)->batch_new(queryBlob, queryParams));
}
VecSimQueryReply *VecSimBatchIterator_Next(VecSimBatchIterator *it, size_t n_results, VecSimQueryReply_Order order) {
    return it->index->batch_next(it, n_results, order);
}
bool VecSimBatchIterator_HasNext(VecSimBatchIterator *it) { return it->returned != it->label_count; }
void VecSimBatchIterator_Reset(VecSimBatchIterator *it) {
    it->scored = false;
    it->returned = 0;
    it->has_cursor = false;
    it->cursor = 0;
    it->seen.clear();
}
void VecSimBatchIterator_Free(VecSimBatchIterator *it) { delete it; }

// ---------------------------------------------------------------------------------- ad-hoc ctx
VecSimAdhocBfCtx *VecSimIndex_AdhocBfCtx_New(VecSimIndex *index, const void *queryBlob) {
    return static_cast<VecSimAdhocBfCtx *>(IX(index)->adhoc_new(queryBlob));
}
void VecSimIndex_AdhocBfCtx_Free(VecSimAdhocBfCtx *ctx) { delete ctx; }
double VecSimIndex_AdhocBfCtx_GetDistanceFrom(VecSimAdhocBfCtx *ctx, size_t label) {
    double d;
    ctx->index->adhoc_distances(ctx, &label, &d, 1);
    return d;
}
void VecSimIndex_AdhocBfCtx_GetExactDistances(VecSimAdhocBfCtx *ctx, const size_t *labels, double *distances_out,
                                              size_t count) {
    ctx->index->adhoc_distances(ctx, labels, distances_out, count);
}

// ---------------------------------------------------------------------------------- replies
size_t VecSimQueryReply_Len(VecSimQueryReply *r) { return r->results.size(); }
VecSimQueryReply_Code VecSimQueryReply_GetCode(VecSimQueryReply *r) { return r->code; }
void VecSimQueryReply_Free(VecSimQueryReply *r) { delete r; }
VecSimQueryReply_Iterator *VecSimQueryReply_GetIterator(VecSimQueryReply *r) { return new VecSimQueryReply_Iterator{r, 0}; }
VecSimQueryResult *VecSimQueryReply_IteratorNext(VecSimQueryReply_Iterator *it) {
    if (it->pos >= it->reply->results.size()) return nullptr;
    return &it->reply->results[it->pos++];
}
bool VecSimQueryReply_IteratorHasNext(VecSimQueryReply_Iterator *it) { return it->pos < it->reply->results.size(); }
void VecSimQueryReply_IteratorReset(VecSimQueryReply_Iterator *it) { it->pos = 0; }
void VecSimQueryReply_IteratorFree(VecSimQueryReply_Iterator *it) { delete it; }
int64_t VecSimQueryResult_GetId(const VecSimQueryResult *item) { return item ? (int64_t)item->id : (int64_t)UINT_MAX; }
double VecSimQueryResult_GetScore(const VecSimQueryResult *item) {
    return item ? item->score : std::numeric_limits<double>::quiet_NaN();
}

// ---------------------------------------------------------------------------------- helpers / info
void VecSim_Normalize(void *blob, size_t dim, VecSimType type) {
    switch (type) {
    case VecSimType_FLOAT32: rsb200::normalize_f32(static_cast<float *>(blob), dim); break;
    case VecSimType_FLOAT16: rsb200::normalize_f16(static_cast<uint16_t *>(blob), dim); break;
    case VecSimType_BFLOAT16: rsb200::normalize_bf16(static_cast<uint16_t *>(blob), dim); break;
    case VecSimType_INT8: rsb200::append_int_norm(static_cast<int8_t *>(blob), dim); break;
    case VecSimType_UINT8: rsb200::append_int_norm(static_cast<uint8_t *>(blob), dim); break;
    default: break;
    }
}
size_t VecSimParams_GetQueryBlobSize(VecSimType type, size_t dim, VecSimMetric metric) { return stored_size(type, dim, metric); }

VecSimIndexBasicInfo VecSimIndex_BasicInfo(VecSimIndex *index) { return IX(index)->basic_info(); }
VecSimIndexStatsInfo VecSimIndex_StatsInfo(VecSimIndex *index) { return IX(index)->stats_info(); }
VecSimIndexDebugInfo VecSimIndex_DebugInfo(VecSimIndex *index) { return IX(index)->debug_info(); }
VecSimDebugInfoIterator *VecSimIndex_DebugInfoIterator(VecSimIndex *index) { return IX(index)->debug_iterator(); }
size_t VecSimDebugInfoIterator_NumberOfFields(VecSimDebugInfoIterator *it) { return it->fields.size(); }
bool VecSimDebugInfoIterator_HasNextField(VecSimDebugInfoIterator *it) { return it->pos < it->fields.size(); }
VecSim_InfoField *VecSimDebugInfoIterator_NextField(VecSimDebugInfoIterator *it) {
    return it->pos < it->fields.size() ? &it->fields[it->pos++] : nullptr;
}
void VecSimDebugInfoIterator_Free(VecSimDebugInfoIterator *it) { delete it; }

void VecSimTieredIndex_GC(VecSimIndex *) {}
void VecSimTieredIndex_AcquireSharedLocks(VecSimIndex *) {}
void VecSimTieredIndex_ReleaseSharedLocks(VecSimIndex *) {}

void VecSim_SetMemoryFunctions(VecSimMemoryFunctions f) { rsb200::globals().mem = f; }
void VecSim_SetTimeoutCallbackFunction(timeoutCallbackFunction cb) { rsb200::globals().timeout_cb.store(cb); }
void VecSim_SetLogCallbackFunction(logCallbackFunction cb) { rsb200::globals().log_cb.store(cb); }
void VecSim_SetWriteMode(VecSimWriteMode) {}
void VecSim_SetTestLogContext(const char *test_name, const char *test_type) {
    auto &g = rsb200::globals();
    std::lock_guard<std::mutex> lk(g.test_ctx_mu);
    g.test_name = test_name ? test_name : "";
    g.test_type = test_type ? test_type : "";
}
void VecSim_UpdateThreadPoolSize(size_t) {}
size_t VecSim_GetSharedMemory(void) { return 0; }

// ---------------------------------------------------------------------------------- extensions
int VecSimB200_TopKQueryBatch(VecSimIndex *index, const void *queryBlobs, size_t qstride, size_t nq, size_t k,
                              VecSimQueryParams *queryParams, size_t *out_labels, double *out_scores) {
    return IX(index)->topk_batch(queryBlobs, qstride, nq, k, queryParams, out_labels, out_scores);
}
int VecSimB200_RangeQueryBatch(VecSimIndex *index, const void *queryBlobs, size_t qstride, size_t nq, const double *radii,
                               VecSimQueryParams *queryParams, VecSimQueryReply_Order order, VecSimQueryReply **replies, uint32_t *out_flags) {
    // the argument checks of VecSimIndex_RangeQuery, for the whole batch before anything is allocated
    if (order != BY_ID && order != BY_SCORE) {
        IX(index)->log("warning", "Possible order values are only 'BY_ID' or 'BY_SCORE'");
        return -1;
    }
    for (size_t i = 0; i < nq; i++)
        if (radii[i] < 0) {
            IX(index)->log("warning", "radius must be non-negative");
            return -1;
        }
    return IX(index)->range_batch(queryBlobs, qstride, nq, radii, queryParams, order, replies, out_flags);
}
int VecSimB200_TopKQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k,
                                    int64_t *d_out_labels, float *d_out_scores, void *stream) {
    return IX(index)->topk_batch_device(d_queries, nq, k, d_out_labels, d_out_scores, static_cast<cudaStream_t>(stream));
}
int VecSimB200_RangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                     VecSimQueryReply_Order order, int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts,
                                     void *stream) {
    return IX(index)->range_batch_device(d_queries, nq, d_radii, cap, order, d_out_labels, d_out_scores, d_out_counts,
                                         static_cast<cudaStream_t>(stream));
}
int VecSimB200_LabelRangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                          VecSimQueryReply_Order order, int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts,
                                          void *stream) {
    return IX(index)->label_range_batch_device(d_queries, nq, d_radii, cap, order, d_out_labels, d_out_scores, d_out_counts,
                                               static_cast<cudaStream_t>(stream));
}
int VecSimB200_AddVectors(VecSimIndex *index, const void *blobs, size_t stride, size_t n, const size_t *labels,
                          size_t label0) {
    return IX(index)->add_bulk(blobs, stride, n, labels, label0);
}
int VecSimB200_AddVectorsDevice(VecSimIndex *index, const void *d_rows, size_t n, size_t label0) {
    return IX(index)->add_bulk_device(d_rows, n, label0);
}
int VecSimB200_Reserve(VecSimIndex *index, size_t rows) { return IX(index)->reserve(rows) ? 0 : -1; }
int VecSimB200_Flush(VecSimIndex *index) { return IX(index)->flush() ? 0 : -1; }
const void *VecSimB200_DeviceRows(VecSimIndex *index, size_t *row_pitch_bytes, size_t *rows) {
    size_t p = 0, r = 0;
    const void *d = IX(index)->device_rows(&p, &r);
    if (row_pitch_bytes) *row_pitch_bytes = p;
    if (rows) *rows = r;
    return d;
}
int VecSimB200_ReadRows(VecSimIndex *index, size_t first_row, size_t n_rows, void *host_dst) {
    return IX(index)->read_rows(first_row, n_rows, host_dst) ? 0 : -1;
}
VecSimB200_Stats VecSimB200_GetStats(VecSimIndex *index, bool reset) { return IX(index)->get_stats(reset); }
int VecSimB200_MergeShardTopK(const float *d_scores, const int64_t *d_labels, size_t G, size_t nq, size_t k,
                              float *d_out_scores, int64_t *d_out_labels, void *stream) {
    return rsb200::launch_merge_shards(d_scores, d_labels, (uint32_t)G, (uint32_t)nq, (uint32_t)k, d_out_scores,
                                       d_out_labels, static_cast<cudaStream_t>(stream), nullptr) == cudaSuccess
               ? 0
               : -1;
}
int VecSimB200_TopKFiltered(VecSimIndex *index, const void *queryBlob, size_t k, const uint32_t *doc_ids, size_t n, int ids_on_device,
                            size_t *out_labels, double *out_scores, size_t *out_count) {
    size_t dummy = 0;
    return IX(index)->topk_filtered(queryBlob, k, doc_ids, n, ids_on_device != 0, out_labels, out_scores, out_count ? out_count : &dummy);
}
int VecSimB200_TopKFilteredBatch(VecSimIndex *index, const void *const *queryBlobs, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                 const size_t *counts, size_t *out_labels, double *out_scores, size_t *out_counts) {
    return IX(index)->topk_filtered_batch(queryBlobs, nq, k, d_doc_ids, counts, out_labels, out_scores, out_counts);
}
int VecSimB200_TopKFilteredBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                       const uint32_t *const *d_counts, const size_t *caps, int64_t *d_out_labels, float *d_out_scores,
                                       uint32_t *d_out_counts, void *stream) {
    return IX(index)->topk_filtered_batch_device(d_queries, nq, k, d_doc_ids, d_counts, caps, d_out_labels, d_out_scores, d_out_counts,
                                                 static_cast<cudaStream_t>(stream));
}
int VecSimB200_HybridTopKBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                     const uint32_t *const *d_counts, const size_t *caps, VecSimQueryParams *queryParams, int64_t *d_out_labels,
                                     float *d_out_scores, uint32_t *d_out_counts, int *out_modes, void *stream) {
    return IX(index)->hybrid_topk_batch_device(d_queries, nq, k, d_doc_ids, d_counts, caps, queryParams, d_out_labels, d_out_scores, d_out_counts,
                                               out_modes, static_cast<cudaStream_t>(stream));
}
int VecSimB200_HybridRangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                           VecSimQueryReply_Order order, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts,
                                           const size_t *caps, VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                           uint32_t *d_out_counts, int *out_modes, void *stream) {
    return IX(index)->hybrid_range_batch_device(d_queries, nq, d_radii, cap, order, d_doc_ids, d_counts, caps, queryParams, d_out_labels,
                                                d_out_scores, d_out_counts, out_modes, static_cast<cudaStream_t>(stream));
}
int VecSimB200_LastBatchPath(VecSimIndex *index) { return IX(index)->last_batch_path(); }
int VecSimB200_LastCoarseShadowBits(VecSimIndex *index) { return IX(index)->last_shadow_bits(); }
void VecSimB200_SetCoarseMode(int mode) { rsb200::set_coarse_mode(mode); }
int VecSimB200_LastCoarseFlags(VecSimIndex *index, uint32_t *out_ok, size_t nq) { return IX(index)->last_coarse_flags(out_ok, nq); }
const char *VecSimB200_Version(void) { return "vecsim_b200 0.1 (sm_90a)"; }

} // extern "C"
