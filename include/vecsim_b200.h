/* vecsim_b200.h — C-ABI of libvecsim_b200.so, the H100-native drop-in for the FLAT (brute-force)
 * slice of the reference's VecSim C API.
 *
 * Every VecSim* entry point below has the same name, argument order, argument meaning, ownership
 * rule and error behaviour as the reference declaration cited next to it (paths relative to
 * /root/reference/deps/VectorSimilarity/src/VecSim/), so RediSearch's callers —
 * src/vector_index.c, src/iterators/hybrid_reader.c, src/document.c:721, src/spec.c:3539 — link
 * against this library unchanged.  Enum values and struct layouts are ABI-identical to
 * vec_sim_common.h / query_results.h (checked by tests/test_abi_layout.py against golden
 * sizeof/offsetof tables taken from the reference headers).  The text of this header is written
 * from scratch; only names and layouts are shared, because they are the ABI.
 *
 * What differs from the reference is where the work happens: the corpus lives in HBM and every
 * distance/top-k computation is a hand-written sm_90a CUDA kernel.  There is no CPU fallback:
 * if no CUDA device is usable VecSimIndex_New returns NULL and logs through the log callback.
 *
 * VecSimB200_* entry points are extensions the reference does not have (batched top-k and range
 * queries, bulk device ingest, shard merge); INTEGRATION.md shows where a RediSearch maintainer would call them.
 */
#ifndef VECSIM_B200_H
#define VECSIM_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Enums — numeric values follow vec_sim_common.h:60-117 and query_results.h:21-26.
 * ---------------------------------------------------------------------------------------------- */
typedef enum {
    VecSimType_FLOAT32 = 0,
    VecSimType_FLOAT64 = 1, /* not on the device path: VecSimIndex_New returns NULL */
    VecSimType_BFLOAT16 = 2,
    VecSimType_FLOAT16 = 3,
    VecSimType_INT8 = 4,
    VecSimType_UINT8 = 5,
    VecSimType_INT32 = 6,
    VecSimType_INT64 = 7
} VecSimType;

typedef enum {
    VecSimAlgo_BF = 0, /* the only algorithm this library implements */
    VecSimAlgo_HNSWLIB = 1,
    VecSimAlgo_TIERED = 2,
    VecSimAlgo_SVS = 3
} VecSimAlgo;

typedef enum { VecSimMetric_L2 = 0, VecSimMetric_IP = 1, VecSimMetric_Cosine = 2 } VecSimMetric;

typedef enum { VecSimOption_AUTO = 0, VecSimOption_ENABLE = 1, VecSimOption_DISABLE = 2 } VecSimOptionMode;
typedef enum { VecSimBool_TRUE = 1, VecSimBool_FALSE = 0, VecSimBool_UNSET = -1 } VecSimBool;

typedef enum { BY_SCORE = 0, BY_ID = 1, BY_SCORE_THEN_ID = 2 } VecSimQueryReply_Order;
typedef enum { VecSim_QueryReply_OK = 0, VecSim_QueryReply_TimedOut = 1 } VecSimQueryReply_Code;

#define VecSim_OK 0
typedef enum {
    VecSimParamResolver_OK = VecSim_OK,
    VecSimParamResolverErr_NullParam,
    VecSimParamResolverErr_AlreadySet,
    VecSimParamResolverErr_UnknownParam,
    VecSimParamResolverErr_BadValue,
    VecSimParamResolverErr_InvalidPolicy_NExits,
    VecSimParamResolverErr_InvalidPolicy_NHybrid,
    VecSimParamResolverErr_InvalidPolicy_NRange,
    VecSimParamResolverErr_InvalidPolicy_AdHoc_With_BatchSize,
    VecSimParamResolverErr_InvalidPolicy_AdHoc_With_EfRuntime
} VecSimResolveCode;

/* vec_sim_common.h:303-319 */
typedef enum {
    EMPTY_MODE = 0,
    STANDARD_KNN,
    HYBRID_ADHOC_BF,
    HYBRID_BATCHES,
    HYBRID_BATCHES_TO_ADHOC_BF,
    RANGE_QUERY
} VecSearchMode;

typedef enum { QUERY_TYPE_NONE = 0, QUERY_TYPE_KNN, QUERY_TYPE_HYBRID, QUERY_TYPE_RANGE } VecsimQueryType;

typedef enum { VecSim_WriteAsync = 0, VecSim_WriteInPlace = 1 } VecSimWriteMode;

typedef enum {
    VecSimSvsQuant_NONE = 0,
    VecSimSvsQuant_Scalar = 1,
    VecSimSvsQuant_4 = 4,
    VecSimSvsQuant_8 = 8,
    VecSimSvsQuant_4x4 = 4 | (4 << 8),
    VecSimSvsQuant_4x8 = 4 | (8 << 8),
    VecSimSvsQuant_4x8_LeanVec = 4 | (8 << 8) | (1 << 16),
    VecSimSvsQuant_8x8_LeanVec = 8 | (8 << 8) | (1 << 16)
} VecSimSvsQuantBits;

#define DEFAULT_BLOCK_SIZE 1024
#define VECSIM_POLICY_ADHOC_BF "adhoc_bf"
#define VECSIM_POLICY_BATCHES "batches"

typedef size_t labelType;      /* == RediSearch t_docId */
typedef unsigned int idType;   /* dense internal row id */

/* ------------------------------------------------------------------------------------------------
 * Parameter structs.  Only BFParams is interpreted; the other arms of the AlgoParams union are
 * declared so that sizeof(VecSimParams) and offsetof(VecSimParams, logCtx) match the reference
 * (vec_sim_common.h:142-268).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const char *name;
    size_t nameLen;
    const char *value;
    size_t valLen;
} VecSimRawParam;

typedef struct {
    VecSimType type;
    size_t dim;
    VecSimMetric metric;
    bool multi;             /* true: one label may own several vectors (JSON multi-value) */
    size_t initialCapacity; /* deprecated upstream; here: rows of HBM to reserve up front */
    size_t blockSize;       /* 0 -> DEFAULT_BLOCK_SIZE; growth granule of the label table */
} BFParams;

typedef struct {
    VecSimType type;
    size_t dim;
    VecSimMetric metric;
    bool multi;
    size_t initialCapacity;
    size_t blockSize;
    size_t M;
    size_t efConstruction;
    size_t efRuntime;
    double epsilon;
} HNSWParams;

typedef struct {
    VecSimType type;
    size_t dim;
    VecSimMetric metric;
    bool multi;
    size_t blockSize;
    VecSimSvsQuantBits quantBits;
    float alpha;
    size_t graph_max_degree;
    size_t construction_window_size;
    size_t max_candidate_pool_size;
    size_t prune_to;
    VecSimOptionMode use_search_history;
    size_t num_threads;
    size_t search_window_size;
    size_t search_buffer_capacity;
    size_t leanvec_dim;
    double epsilon;
} SVSParams;

typedef struct AsyncJob AsyncJob;
typedef void (*JobCallback)(AsyncJob *);
typedef int (*SubmitCB)(void *job_queue, void *index_ctx, AsyncJob **jobs, JobCallback *CBs, size_t jobs_len);
typedef struct VecSimParams VecSimParams;

typedef struct { size_t swapJobThreshold; } TieredHNSWParams;
typedef struct { char _placeholder; } TieredHNSWDiskParams;
typedef struct {
    size_t trainingTriggerThreshold;
    size_t updateTriggerThreshold;
    size_t updateJobWaitTime;
} TieredSVSParams;

typedef struct {
    void *jobQueue;
    void *jobQueueCtx;
    SubmitCB submitCb;
    size_t flatBufferLimit;
    VecSimParams *primaryIndexParams;
    union {
        TieredHNSWParams tieredHnswParams;
        TieredSVSParams tieredSVSParams;
        TieredHNSWDiskParams tieredHnswDiskParams;
    } specificParams;
} TieredIndexParams;

typedef union {
    HNSWParams hnswParams;
    BFParams bfParams;
    TieredIndexParams tieredParams;
    SVSParams svsParams;
} AlgoParams;

struct VecSimParams {
    VecSimAlgo algo; /* must be VecSimAlgo_BF */
    AlgoParams algoParams;
    void *logCtx; /* handed back as the first argument of the log callback */
};

/* Runtime (per query) parameters, vec_sim_common.h:283-338.  FLAT reads batchSize, searchMode and
 * timeoutCtx only. */
typedef struct { size_t efRuntime; double epsilon; } HNSWRuntimeParams;
typedef struct { size_t efRuntime; double epsilon; VecSimBool shouldRerank; } HNSWDiskRuntimeParams;
typedef struct {
    size_t windowSize;
    size_t bufferCapacity;
    VecSimOptionMode searchHistory;
    double epsilon;
} SVSRuntimeParams;

typedef struct {
    union {
        HNSWRuntimeParams hnswRuntimeParams;
        HNSWDiskRuntimeParams hnswDiskRuntimeParams;
        SVSRuntimeParams svsRuntimeParams;
    };
    size_t batchSize;
    VecSearchMode searchMode;
    void *timeoutCtx; /* passed to the timeout callback between kernel launches */
} VecSimQueryParams;

/* vec_sim_common.h:343-360 */
typedef struct {
    VecSimAlgo algo;
    VecSimMetric metric;
    VecSimType type;
    bool isMulti;
    bool isTiered;
    bool isDisk;
    size_t blockSize;
    size_t dim;
} VecSimIndexBasicInfo;

typedef struct {
    size_t memory; /* host bytes + HBM bytes owned by the index */
    size_t numberOfMarkedDeleted;
    size_t directHNSWInsertions;
    size_t flatBufferSize;
} VecSimIndexStatsInfo;

/* VecSimIndexDebugInfo (vec_sim_common.h:372-457): returned BY VALUE by VecSimIndex_DebugInfo, so the whole union has to keep
 * the reference's size and member offsets even though a FLAT index only fills commonInfo and bfInfo. */
typedef struct {
    VecSimIndexBasicInfo basicInfo;
    size_t indexSize;       /* current count of vectors */
    size_t indexLabelCount; /* current unique count of labels */
    uint64_t memory;
    VecSearchMode lastMode; /* the mode in which the last query ran */
} CommonInfo;
typedef struct { size_t M, efConstruction, efRuntime; double epsilon; size_t max_level, entrypoint, visitedNodesPoolSize,
                 numberOfMarkedDeletedNodes; } hnswInfoStruct;
typedef struct { char dummy; } bfInfoStruct;
typedef struct {
    VecSimSvsQuantBits quantBits;
    float alpha;
    size_t graphMaxDegree, constructionWindowSize, maxCandidatePoolSize, pruneTo;
    bool useSearchHistory;
    size_t numThreads, lastReservedThreads, numberOfMarkedDeletedNodes, searchWindowSize, searchBufferCapacity, leanvecDim;
    double epsilon;
} svsInfoStruct;
typedef struct HnswTieredInfo { size_t pendingSwapJobsThreshold; } HnswTieredInfo;
typedef struct SvsTieredInfo { size_t trainingTriggerThreshold, updateTriggerThreshold, updateJobWaitTime; bool indexUpdateScheduled; } SvsTieredInfo;
typedef struct {
    union { hnswInfoStruct hnswInfo; svsInfoStruct svsInfo; } backendInfo;
    union { HnswTieredInfo hnswTieredInfo; SvsTieredInfo svsTieredInfo; } specificTieredBackendInfo;
    CommonInfo backendCommonInfo;
    CommonInfo frontendCommonInfo;
    bfInfoStruct bfInfo;
    uint64_t management_layer_memory;
    VecSimBool backgroundIndexing;
    size_t bufferLimit;
} tieredInfoStruct;
typedef struct {
    CommonInfo commonInfo;
    union {
        bfInfoStruct bfInfo;
        hnswInfoStruct hnswInfo;
        svsInfoStruct svsInfo;
        tieredInfoStruct tieredInfo;
    };
} VecSimIndexDebugInfo;

/* Debug-info iterator (info_iterator.h:17-44).  Fields reported for FLAT: ALGORITHM, TYPE,
 * DIMENSION, METRIC, IS_MULTI_VALUE, IS_DISK, INDEX_SIZE, INDEX_LABEL_COUNT, MEMORY,
 * LAST_SEARCH_MODE, BLOCK_SIZE (brute_force.h:327-365). */
typedef struct VecSimDebugInfoIterator VecSimDebugInfoIterator;
typedef enum { INFOFIELD_STRING, INFOFIELD_INT64, INFOFIELD_UINT64, INFOFIELD_FLOAT64, INFOFIELD_ITERATOR } VecSim_InfoFieldType;
typedef union {
    double floatingPointValue;
    int64_t integerValue;
    uint64_t uintegerValue;
    const char *stringValue;
    VecSimDebugInfoIterator *iteratorValue;
} FieldValue;
typedef struct {
    const char *fieldName;
    VecSim_InfoFieldType fieldType;
    FieldValue fieldValue;
} VecSim_InfoField;

typedef void *(*allocFn)(size_t n);
typedef void *(*callocFn)(size_t nelem, size_t elemsz);
typedef void *(*reallocFn)(void *p, size_t n);
typedef void (*freeFn)(void *p);
typedef struct {
    allocFn allocFunction;
    callocFn callocFunction;
    reallocFn reallocFunction;
    freeFn freeFunction;
} VecSimMemoryFunctions;

typedef int (*timeoutCallbackFunction)(void *ctx); /* non-zero = expired */
typedef void (*logCallbackFunction)(void *ctx, const char *level, const char *message);

/* Opaque handles. */
typedef struct VecSimIndexInterface VecSimIndex;
typedef struct VecSimQueryResult VecSimQueryResult;
typedef struct VecSimQueryReply VecSimQueryReply;
typedef struct VecSimQueryReply_Iterator VecSimQueryReply_Iterator;
typedef struct VecSimBatchIterator VecSimBatchIterator;
typedef struct VecSimAdhocBfCtx VecSimAdhocBfCtx;

/* ------------------------------------------------------------------------------------------------
 * Index lifetime and mutation  (vec_sim.h:28-71, vec_sim.cpp:213-236)
 * ---------------------------------------------------------------------------------------------- */
/* vec_sim.h:28.  NULL if params->algo != BF, the type is unsupported, or no CUDA device. */
VecSimIndex *VecSimIndex_New(const VecSimParams *params);
/* vec_sim.h:36,49: host-side estimate, same formula family as brute_force_factory.cpp:96-135. */
size_t VecSimIndex_EstimateInitialSize(const VecSimParams *params);
size_t VecSimIndex_EstimateElementSize(const VecSimParams *params);
/* vec_sim.h:55 */
void VecSimIndex_Free(VecSimIndex *index);
/* vec_sim.h:65.  Blob is copied (cosine: normalised copy, preprocessors.h:49-146).  Single-value
 * index: an existing label is overwritten in place and 0 is returned, else 1. */
int VecSimIndex_AddVector(VecSimIndex *index, const void *blob, size_t label);
/* vec_sim.h:73.  Swap-delete: the last row moves into the hole (brute_force.h:196-224). */
int VecSimIndex_DeleteVector(VecSimIndex *index, size_t label);
/* vec_sim.h:116 */
size_t VecSimIndex_IndexSize(VecSimIndex *index);

/* ------------------------------------------------------------------------------------------------
 * Queries
 * ---------------------------------------------------------------------------------------------- */
/* vec_sim.h:143 / brute_force.h:243-291.  k nearest by (score asc, label asc); k==0 -> empty;
 * k>size -> size results.  order BY_ID sorts the reply by label (vec_sim.cpp:353-355). */
VecSimQueryReply *VecSimIndex_TopKQuery(VecSimIndex *index, const void *queryBlob, size_t k,
                                        VecSimQueryParams *queryParams, VecSimQueryReply_Order order);
/* vec_sim.h:159 / brute_force.h:293-326.  All rows with score <= (float)radius.  Returns NULL and
 * logs for radius < 0 or an order other than BY_ID/BY_SCORE (the reference throws,
 * vec_sim.cpp:362-367). */
VecSimQueryReply *VecSimIndex_RangeQuery(VecSimIndex *index, const void *queryBlob, double radius,
                                         VecSimQueryParams *queryParams, VecSimQueryReply_Order order);
/* vec_sim.h:91 / brute_force_single.h:200-212.  blob must already be normalised for cosine.
 * NaN if the label is absent; multi-value: min over the label's vectors. */
double VecSimIndex_GetDistanceFrom_Unsafe(VecSimIndex *index, size_t label, const void *blob);
/* vec_sim.h:229 / brute_force.h:380-451 (decision tree reproduced exactly; sets lastMode). */
bool VecSimIndex_PreferAdHocSearch(VecSimIndex *index, size_t subsetSize, size_t k, bool initial_check);
/* vec_sim.h:128 / vec_sim.cpp:270-343 */
VecSimResolveCode VecSimIndex_ResolveParams(VecSimIndex *index, VecSimRawParam *rparams, int paramNum,
                                            VecSimQueryParams *qparams, VecsimQueryType query_type);

/* Batch iterator, vec_sim.h:205 + query_results.h:115-138 / bf_batch_iterator.h.  The first Next
 * runs one full scan into an HBM score array; every Next returns the next-best n_results. */
VecSimBatchIterator *VecSimBatchIterator_New(VecSimIndex *index, const void *queryBlob,
                                             VecSimQueryParams *queryParams);
VecSimQueryReply *VecSimBatchIterator_Next(VecSimBatchIterator *iterator, size_t n_results,
                                           VecSimQueryReply_Order order);
bool VecSimBatchIterator_HasNext(VecSimBatchIterator *iterator);
void VecSimBatchIterator_Reset(VecSimBatchIterator *iterator);
void VecSimBatchIterator_Free(VecSimBatchIterator *iterator);

/* Ad-hoc context, vec_sim.h:247-281.  The reference returns NULL for RAM indexes
 * (vec_sim_interface.h:203); here it is implemented because a per-label device round trip is the
 * wrong shape for a GPU: _New uploads the (normalised) query once, _GetExactDistances computes a
 * whole label batch with one gather kernel. */
VecSimAdhocBfCtx *VecSimIndex_AdhocBfCtx_New(VecSimIndex *index, const void *queryBlob);
void VecSimIndex_AdhocBfCtx_Free(VecSimAdhocBfCtx *ctx);
double VecSimIndex_AdhocBfCtx_GetDistanceFrom(VecSimAdhocBfCtx *ctx, size_t label);
void VecSimIndex_AdhocBfCtx_GetExactDistances(VecSimAdhocBfCtx *ctx, const size_t *labels,
                                              double *distances_out, size_t count);

/* Replies, query_results.h:31-101 / query_results.cpp:23-73. */
size_t VecSimQueryReply_Len(VecSimQueryReply *reply);
VecSimQueryReply_Code VecSimQueryReply_GetCode(VecSimQueryReply *reply);
void VecSimQueryReply_Free(VecSimQueryReply *reply);
VecSimQueryReply_Iterator *VecSimQueryReply_GetIterator(VecSimQueryReply *reply);
VecSimQueryResult *VecSimQueryReply_IteratorNext(VecSimQueryReply_Iterator *iterator);
bool VecSimQueryReply_IteratorHasNext(VecSimQueryReply_Iterator *iterator);
void VecSimQueryReply_IteratorReset(VecSimQueryReply_Iterator *iterator);
void VecSimQueryReply_IteratorFree(VecSimQueryReply_Iterator *iterator);
int64_t VecSimQueryResult_GetId(const VecSimQueryResult *item);   /* NULL -> INVALID_ID (UINT_MAX) */
double VecSimQueryResult_GetScore(const VecSimQueryResult *item); /* NULL -> NaN */

/* ------------------------------------------------------------------------------------------------
 * Blob helpers, info, process-wide hooks
 * ---------------------------------------------------------------------------------------------- */
/* vec_sim.h:100 / normalize_naive.h:23-88 (host arithmetic, bit-identical to the reference). */
void VecSim_Normalize(void *blob, size_t dim, VecSimType type);
/* vec_sim.h:113: dim*sizeof(type) (+4 for INT8/UINT8 cosine). */
size_t VecSimParams_GetQueryBlobSize(VecSimType type, size_t dim, VecSimMetric metric);

VecSimIndexBasicInfo VecSimIndex_BasicInfo(VecSimIndex *index);               /* vec_sim.h:178 */
VecSimIndexStatsInfo VecSimIndex_StatsInfo(VecSimIndex *index);               /* vec_sim.h:185 */
VecSimIndexDebugInfo VecSimIndex_DebugInfo(VecSimIndex *index);               /* vec_sim.h:170; FLAT: BruteForceIndex::debugInfo, brute_force.h:318-325 */
VecSimDebugInfoIterator *VecSimIndex_DebugInfoIterator(VecSimIndex *index);   /* vec_sim.h:193 */
size_t VecSimDebugInfoIterator_NumberOfFields(VecSimDebugInfoIterator *it);   /* info_iterator.h:50 */
bool VecSimDebugInfoIterator_HasNextField(VecSimDebugInfoIterator *it);
VecSim_InfoField *VecSimDebugInfoIterator_NextField(VecSimDebugInfoIterator *it);
void VecSimDebugInfoIterator_Free(VecSimDebugInfoIterator *it);

void VecSimTieredIndex_GC(VecSimIndex *index);                    /* no-op for FLAT, vec_sim.h:211 */
void VecSimTieredIndex_AcquireSharedLocks(VecSimIndex *index);    /* no-op, vec_sim.h:237 */
void VecSimTieredIndex_ReleaseSharedLocks(VecSimIndex *index);    /* no-op, vec_sim.h:239 */

void VecSim_SetMemoryFunctions(VecSimMemoryFunctions memoryfunctions);   /* vec_sim.h:288 */
void VecSim_SetTimeoutCallbackFunction(timeoutCallbackFunction callback); /* vec_sim.h:295 */
void VecSim_SetLogCallbackFunction(logCallbackFunction callback);        /* vec_sim.h:302 */
void VecSim_SetWriteMode(VecSimWriteMode mode);                           /* no-op, vec_sim.h:320 */
void VecSim_SetTestLogContext(const char *test_name, const char *test_type); /* vec_sim.h:303: names the log file of the reference's
                                                                                 test logger; kept and shown by the default log sink */
void VecSim_UpdateThreadPoolSize(size_t new_size);                        /* no-op, vec_sim.h:330 */
size_t VecSim_GetSharedMemory(void);                                      /* 0,    vec_sim.h:338 */

/* ------------------------------------------------------------------------------------------------
 * Device extensions (no reference counterpart)
 * ---------------------------------------------------------------------------------------------- */
/* nq queries in one corpus pass.  queryBlobs: nq host blobs, qstride bytes apart.  Results are
 * written to out_labels / out_scores ([nq][k], row-major, ascending (score,label)); entries past
 * the number of hits carry label SIZE_MAX and score NaN.  A multi-value index answers the k best
 * labels, each scored by its best row, as VecSimIndex_TopKQuery does (k <= 128: a tensor-core row route
 * + label stage, queries it cannot prove and corpora of >= 65536 rows no such route serves one at a
 * time; the label-aware exact scan below that size; k > 128: one query at a time).  int8 / uint8 corpora with inner
 * product, cosine or L2 (nq >= 16, >= 65536 rows, dim % 16 == 0, 32 <= dim <= 2048, k <= 128, coarse mode 1 or 2) take the
 * s8 / u8 tensor-core route, bit-exact with the reference (ids, score bits and tie order).  Single-value indexes with
 * 128 < min(k, rows) <= 1024: batches the fp32 route serves (fp32, coarse mode 1 with the fixed bound, nq >= 16, >= 65536
 * rows, dim % 8 == 0, 32..1024, rows inside the fp16 range) run as one batch, the queries it cannot prove finishing on the
 * exact batched top-k on the device (DESIGN.md §4.5); every other such batch, and k > 1024, one query at a time.  Returns
 * VecSim_QueryReply_OK / _TimedOut, or -1 on a CUDA failure. */
int VecSimB200_TopKQueryBatch(VecSimIndex *index, const void *queryBlobs, size_t qstride, size_t nq,
                              size_t k, VecSimQueryParams *queryParams, size_t *out_labels,
                              double *out_scores);
/* Same, but queries and results are DEVICE pointers (fp/int data as the index type; labels are
 * int64, -1 for empty entries, scores float).  Nothing crosses PCIe; the call only enqueues on `stream`
 * (a cudaStream_t cast to void*, NULL = the index's own stream) and returns.  Single-value indexes: k <= 1024 (above 128
 * the fp32 route where it applies, otherwise the exact batched top-k on the device, DESIGN.md §4.5); multi-value indexes:
 * k <= 128; -1 for a larger k. */
int VecSimB200_TopKQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k,
                                    int64_t *d_out_labels, float *d_out_scores, void *stream);
/* nq range queries in one call.  replies[i] receives exactly what
 * VecSimIndex_RangeQuery(index, queryBlobs + i*qstride, radii[i], queryParams, order) would return
 * (same labels, same float scores, same order); the caller frees each with VecSimQueryReply_Free.
 * Single-value fp32 indexes of >= 65536 rows (dim % 8 == 0, 32..1024; coarse mode 1) answer a batch of
 * >= 16 queries with one tensor-core pass over the fp16 shadow, exact rescoring and a per-query
 * completeness proof; every other query is answered by the exact scan, one query at a time.
 * out_flags (nullable, [nq]): 1 = answered by the tensor-core route, 0 = by the exact scan.
 * Returns VecSim_QueryReply_OK / _TimedOut (the timeout callback fired: the replies carry that code,
 * those answered before it fired keep their results, as VecSimIndex_RangeQuery's do); -1 for an order other
 * than BY_ID / BY_SCORE, a negative radius (no reply is allocated, the index logs a warning, as
 * VecSimIndex_RangeQuery does) or a CUDA failure. */
int VecSimB200_RangeQueryBatch(VecSimIndex *index, const void *queryBlobs, size_t qstride, size_t nq,
                               const double *radii, VecSimQueryParams *queryParams,
                               VecSimQueryReply_Order order, VecSimQueryReply **replies, uint32_t *out_flags);
/* nq range queries with DEVICE pointers end to end (DESIGN.md §4.11).  d_queries: stored-form blobs as for
 * VecSimB200_TopKQueryBatchDevice; d_radii: one float per query, in DistType.  Query i's answer is every row with
 * score <= d_radii[i] (a float compare: -0.0 == +0.0, a NaN score never passes, a NaN radius keeps nothing).  A negative
 * radius is answered as given (inner-product distances can be negative), where VecSimB200_RangeQueryBatch refuses it.
 * d_out_counts[i] = the true number of hits, even past cap.  count <= cap: entries [0, count) of row i of d_out_labels /
 * d_out_scores ([nq][cap], int64 / float) hold them, BY_SCORE ordered by (score, label), BY_ID by label, as
 * VecSimIndex_RangeQuery orders its reply; the rest of the row is label -1, score NaN.  count > cap: the whole row is -1 / NaN
 * (re-issue the query with a larger cap, or use VecSimB200_RangeQueryBatch).
 * Routes: single-value fp32 batches the fp32 route of VecSimB200_RangeQueryBatch serves take it; int8 / uint8 batches of
 * >= 16 queries (dim % 16 == 0, 32..2048, >= 65536 rows, coarse mode 1 or 2, VECSIM_B200_FIXED not 0) take a fixed-radius
 * pass on the integer tensor cores, whose distances are the reference's; fp16 / bf16 inner-product or cosine batches of >= 16
 * queries (dim % 8 == 0, 32..1024, >= 65536 rows, coarse mode 1 or 2, VECSIM_B200_FIXED not 0, a finite largest row norm)
 * take the direct 16-bit pass with the bound radius + eps16_q and CUDA-core rescoring, which gives the exact scan's bits; every
 * other query (fp16 / bf16 L2, a query with an inf or NaN component, a NaN or infinite radius), and every query a route cannot
 * complete, takes the exact scan on the device.  The call only enqueues on `stream` (NULL = the legacy default stream); the
 * host waits only for the first build of the fp16 shadow / the int32 |row|^2 table of 8-bit L2 indexes / the |row|^2 table of
 * 16-bit indexes or their refresh after mutations.  After a synchronise, VecSimB200_LastCoarseFlags gives 1 per query a
 * tensor-core route answered and 0 per query the exact scan answered; VecSimB200_LastBatchPath is 1 (fp32 route), 2 (8-bit or
 * 16-bit route) or 0 (exact scan only).  The scratch is that of VecSimB200_TopKQueryBatchDevice.
 * Returns 0 (0 with nothing enqueued for nq == 0); -1 for a multi-value index, cap == 0 or cap > 4096, an order other than
 * BY_ID / BY_SCORE, or a CUDA failure. */
int VecSimB200_RangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                     VecSimQueryReply_Order order, int64_t *d_out_labels, float *d_out_scores,
                                     uint32_t *d_out_counts, void *stream);
/* nq range queries, device pointers end to end, answered per LABEL as VecSimIndex_RangeQuery answers them on any FLAT index
 * (DESIGN.md §4.12).  Arguments, outputs, cap rule, orders, stream, host waits and routes (fp32, 8-bit and 16-bit) as
 * VecSimB200_RangeQueryBatchDevice.
 * Multi-value index: a label is in query i's answer iff one of its rows has score <= d_radii[i] (float compare; a NaN score
 * never passes); its score is the smallest such row score; d_out_counts[i] is the true number of such LABELS.  The first call
 * after a mutation also waits for the rebuild of the label tables.  After a synchronise, VecSimB200_LastCoarseFlags gives 1 per
 * query a route answered, 3 per query a route proved whose hit rows were too many to fold (more than 4096; the exact scan
 * answered it) and 0 per query the exact scan answered.  Single-value index: exactly VecSimB200_RangeQueryBatchDevice.
 * Returns 0; -1 as VecSimB200_RangeQueryBatchDevice (except for multi-value indexes); -2, before anything is enqueued, for a
 * multi-value index whose labels are too sparse for the dense table (the rule of VecSimB200_TopKFiltered: a label >= 2^32 - 1
 * or beyond 4 x rows + 2^24). */
int VecSimB200_LabelRangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                          VecSimQueryReply_Order order, int64_t *d_out_labels, float *d_out_scores,
                                          uint32_t *d_out_counts, void *stream);
/* Bulk ingest of n host blobs (stride bytes apart) with labels[i] (NULL -> label0+i).  Equivalent
 * to n VecSimIndex_AddVector calls on fresh labels, with one H2D transfer per staging buffer. */
int VecSimB200_AddVectors(VecSimIndex *index, const void *blobs, size_t stride, size_t n,
                          const size_t *labels, size_t label0);
/* Bulk ingest of n rows that are already in device memory in stored form (cosine: already
 * normalised; int8/uint8 cosine: norm appended), row pitch = stored row size. */
int VecSimB200_AddVectorsDevice(VecSimIndex *index, const void *d_rows, size_t n, size_t label0);
/* Make sure HBM for `rows` vectors is reserved (avoids regrowth copies). */
int VecSimB200_Reserve(VecSimIndex *index, size_t rows);
/* Block until all staged rows are resident in HBM. */
int VecSimB200_Flush(VecSimIndex *index);
/* Device pointer / pitch of the resident corpus (for tests and the bench's roofline maths). */
const void *VecSimB200_DeviceRows(VecSimIndex *index, size_t *row_pitch_bytes, size_t *rows);
/* Launch statistics since the last call with reset=true: number of this library's kernels
 * launched, and device microseconds of the dominant scan kernel measured with CUDA events on the
 * launching stream. */
typedef struct {
    uint64_t kernel_launches;
    uint64_t scan_launches;
    double scan_device_us;
    uint64_t scan_bytes; /* algorithmic bytes the timed scan launches covered */
} VecSimB200_Stats;
VecSimB200_Stats VecSimB200_GetStats(VecSimIndex *index, bool reset);
/* Copy stored-form rows [first_row, first_row + n_rows) (internal row order, after the storage preprocessor: what
 * DataBlocksContainer holds in the reference) from HBM into a tightly packed host buffer of n_rows * stored-size bytes.
 * For persistence (RDB save) and for checking the device's corpus against a CPU scan.  0 / -1. */
int VecSimB200_ReadRows(VecSimIndex *index, size_t first_row, size_t n_rows, void *host_dst);
/* G-way merge of per-shard top-k lists (the coordinator's knnPostProcess, src/module.c:3139-3176,
 * comparator VecSim utils/query_result_utils.h:19-23), on device: in = [G][nq][k] gathered
 * (score,label) pairs, out = [nq][k]. */
int VecSimB200_MergeShardTopK(const float *d_scores, const int64_t *d_labels, size_t G, size_t nq,
                              size_t k, float *d_out_scores, int64_t *d_out_labels, void *stream);
/* ---- sharded KNN across GPUs, the exchange inside the library (SURVEY.md §8e) -------------------------------------------
 * One process per GPU, every process holds one row shard in its own VecSimIndex.  A query batch is answered by: local scan
 * of the shard -> ONE ncclAllGather of the packed per-shard top-k (labels + scores of a rank in one block) over NVLink ->
 * G-way merge on device by (score, label) — the coordinator's knnPostProcess, src/module.c:3139-3176, comparator
 * VS/utils/query_result_utils.h:19-23.  NCCL is bound at run time (dlopen "libnccl.so.2", or VECSIM_B200_NCCL_LIB), so
 * single-GPU users never load it.  Bootstrap like any NCCL program: rank 0 calls _UniqueId, ships the 128 bytes to the
 * other ranks over whatever control channel the host has (RediSearch: the cluster bus), every rank calls _New. */
typedef struct VecSimB200_ShardGroup VecSimB200_ShardGroup;
/* The exchange block of one shard: [labels int64 x nq*k][scores float x nq*k] padded to 16 bytes; and the merge of G such
 * blocks laid out rank-major (what an all-gather leaves) — for hosts that move the blocks with their own transport. */
size_t VecSimB200_ShardBlockBytes(size_t nq, size_t k);
int VecSimB200_MergeShardBlocks(const void *d_blocks, size_t G, size_t nq, size_t k, float *d_out_scores, int64_t *d_out_labels,
                                void *stream);
int VecSimB200_ShardGroup_UniqueId(void *out128);                                        /* 0 = ok */
VecSimB200_ShardGroup *VecSimB200_ShardGroup_New(const void *id128, int rank, int world); /* collective; NULL on error */
void VecSimB200_ShardGroup_Free(VecSimB200_ShardGroup *g);
int VecSimB200_ShardGroup_Rank(const VecSimB200_ShardGroup *g);
int VecSimB200_ShardGroup_Size(const VecSimB200_ShardGroup *g);
/* Collective, enqueued on `stream`, nothing synchronised: d_queries = nq stored-form (normalised) query blobs on this
 * rank's device; every rank receives the merged [nq][k] labels (int64, -1 = empty) and distances.  k as in
 * VecSimB200_TopKQueryBatchDevice: up to 1024 on single-value shards, 128 on multi-value shards; -1 beyond. */
int VecSimB200_ShardGroup_TopKBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq, size_t k,
                                          int64_t *d_out_labels, float *d_out_scores, void *stream);
/* Collective, host buffers end to end (raw query blobs in as for VecSimIndex_TopKQuery; H2D, shard scan, all-gather,
 * merge, D2H inside the call).  Empty slots: label SIZE_MAX, score NaN.  The same limits on k.  Returns 0 / -1. */
int VecSimB200_ShardGroup_TopKBatch(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *queryBlobs, size_t qstride, size_t nq,
                                    size_t k, size_t *out_labels, double *out_scores);
/* ---- sharded filtered KNN, range and filtered range batches (DESIGN.md §6.1) ----------------------------------------------------
 * The counted exchange block of one rank: [labels int64 x nq*w][scores float x nq*w][counts u32 x nq], padded to 16 bytes.  Row i and
 * counts[i] are what the rank's local device call wrote for query i: KNN, the entries written (<= w); range, the true number of hits
 * (past w the row is all -1); UINT32_MAX, the rank could not answer.  Blocks are rank-major after an all-gather. */
size_t VecSimB200_ShardListBlockBytes(size_t nq, size_t w);
/* Merge of G such blocks on the device into [nq][w] labels / scores and [nq] counts, enqueued on `stream` (NULL = the legacy default
 * stream).  range == 0 (top-w, BY_SCORE only): the first w entries of the union by (score, label), count = min(w, sum of counts).
 * range == 1: total = the sum of the counts (saturating at UINT32_MAX); total > w gives the row all -1 / NaN with count = total (the cap
 * rule of the range calls), otherwise the union in the local calls' order (BY_SCORE: (score, label); BY_ID: label), count = total.  A
 * rank with count UINT32_MAX makes the row empty with count UINT32_MAX.  Entries sort by the key the local calls sort by (-0.0 ties
 * +0.0, ties break by label, then by rank) and keep their score bits, so merging the shards of a corpus whose labels each live on one
 * shard gives, bit for bit, the rows the local call gives on one index holding the whole corpus.  Runs must be sorted, as every local
 * call writes them.  One launch, O(G m log m) per query for runs of m entries.
 * Returns 0; -1, before any CUDA call, for G == 0, w == 0 or w > 4096, nq > 2^31, range not 0 / 1, an order other than BY_SCORE /
 * BY_ID, BY_ID with range == 0; -1 for a CUDA failure. */
int VecSimB200_MergeShardListBlocks(const void *d_blocks, size_t G, size_t nq, size_t w, int range, VecSimQueryReply_Order order,
                                    int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts, void *stream);
/* Collectives: this rank's local call (VecSimB200_HybridTopKBatchDevice, VecSimB200_LabelRangeQueryBatchDevice,
 * VecSimB200_HybridRangeQueryBatchDevice) writes straight into the group's send block, ONE ncclAllGather, the list merge; every
 * rank receives the merged rows and counts.  Arguments mean what they mean in the local call; the filters are THIS rank's docIds (its
 * slice of each posting list, cut at the shard boundaries), and out_modes / VecSimB200_LastCoarseFlags report this rank's routes.
 * Shards hold disjoint labels (a multi-value label's rows all on one shard): the merged rows, scores and counts are then bit-equal to
 * the local call on one index holding every shard's rows, with the union of the filters.  world == 1: the call IS the local call (no
 * NCCL is loaded).  Launches: the local call's + 1 all-gather + 1 merge, enqueued on `stream`; the host waits for nothing beyond what
 * the local call waits for.  The group's blocks grow under its mutex.  An empty shard takes part with counts 0.
 * Failures never leave a rank waiting in the all-gather: refusals from the shared arguments (k > 1024, cap outside 1..4096, an order
 * other than BY_SCORE / BY_ID, a bad searchMode, nq > 2^31) return -1 on every rank before anything is enqueued; a refusal of the
 * local call itself (-2 for labels too sparse for the docId table or a cap beyond the 32-bit range, -1 for a failed flush) still
 * takes part with a block of counts UINT32_MAX and returns its code, and every rank's merged rows come out empty with count
 * UINT32_MAX.  A CUDA or NCCL failure after the enqueue is -1. */
int VecSimB200_ShardGroup_HybridTopKBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq, size_t k,
                                                const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                                VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                                uint32_t *d_out_counts, int *out_modes, void *stream);
int VecSimB200_ShardGroup_RangeQueryBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq,
                                                const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_out_labels,
                                                float *d_out_scores, uint32_t *d_out_counts, void *stream);
int VecSimB200_ShardGroup_HybridRangeQueryBatchDevice(VecSimB200_ShardGroup *g, VecSimIndex *shard, const void *d_queries, size_t nq,
                                                      const float *d_radii, size_t cap, VecSimQueryReply_Order order,
                                                      const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                                      VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                                      uint32_t *d_out_counts, int *out_modes, void *stream);
/* The whole HybridIterator state machine of src/iterators/hybrid_reader.c in one call: mode choice (:668-691:
 * VecSimIndex_PreferAdHocSearch on the child's estimate unless qp->searchMode forces a policy), HYBRID_BATCHES with the
 * reference's batch-size formula (:400-404), the alternating merge of each BY_ID batch with the child (:140-169) and the
 * policy review that may restart in ad-hoc mode (:346-370, :430-438), and HYBRID_ADHOC_BF (:289-335) served by ONE fused
 * device call over the drained child docIds instead of a GetDistanceFrom round trip per document.  child_iterator: any
 * object with the reference's QueryIterator vtable (iterator_api.h:46-151) — a device AND / OR result or a host iterator; it
 * is NOT freed.  The k best are kept in the reference's heap order (cmpVecSimResByScore :35-44) and written ordered by
 * (score, docId).  *out_mode = VecSearchMode the query ended in (also VecSimIndex's LAST_SEARCH_MODE), *out_iterations =
 * batches run.  Multi-value indexes are served in every mode (ad-hoc mode through VecSimB200_TopKFiltered's fold).
 * Returns a VecSimQueryReply_Code, or -1 (also for labels too sparse for ad-hoc mode).  Exact score ties at the k-th place in ad-hoc mode resolve towards
 * the smaller docId (the reference's min-max heap evicts the smaller docId among tied worst entries). */
int VecSimB200_HybridTopK(VecSimIndex *index, const void *queryBlob, size_t k, void *child_iterator, VecSimQueryParams *queryParams,
                          size_t *out_labels, double *out_scores, size_t *out_count, int *out_mode, size_t *out_iterations);
/* Hybrid "filter AND KNN" in ad-hoc mode, fused: what HybridIterator does in HYBRID_ADHOC_BF mode
 * (src/iterators/hybrid_reader.c:289-335: read the child iterator's docIds in ascending order, GetDistanceFrom each,
 * keep the k best in a heap with strict `<` admission, skip NaN = deleted) — in one call.  doc_ids: the filter's
 * ascending docIds (= vector labels), on the host or on the device (ids_on_device != 0, e.g.
 * II_ResultSet_DeviceDocIds of the filter's AND/OR).  Writes up to k (label, distance) pairs ordered by
 * (distance asc, docId asc) and their number.  Multi-value indexes are served: a docId's distance is getDistanceFrom_Unsafe's
 * fold over its rows (brute_force_multi.h:224-241, dist = (dist < d) ? dist : d from +inf in insertion order, so a NaN in the
 * label's last row makes it NaN and the docId is skipped).  Returns 0; -2 if the labels are too sparse for the dense docId ->
 * rows table (a label >= 2^32 - 1, or beyond 4 x rows + 2^24) or n exceeds the 32-bit id range — the caller then stays on
 * VecSimIndex_GetDistanceFrom_Unsafe. */
int VecSimB200_TopKFiltered(VecSimIndex *index, const void *queryBlob, size_t k, const uint32_t *doc_ids, size_t n, int ids_on_device,
                            size_t *out_labels, double *out_scores, size_t *out_count);
/* The same for nq hybrid queries in one call (k <= 128): queryBlobs[i] with the DEVICE-resident ascending docId list
 * d_doc_ids[i] of counts[i] entries (its filter's AND / OR result).  Every query's kernel chain is enqueued on its own stream
 * before anything is waited for.  out_labels / out_scores are [nq][k], out_counts[i] the entries written for query i.
 * Multi-value indexes as in VecSimB200_TopKFiltered.  Returns 0; -2 for sparse labels, k > 128 or a list beyond the 32-bit id
 * range. */
int VecSimB200_TopKFilteredBatch(VecSimIndex *index, const void *const *queryBlobs, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                 const size_t *counts, size_t *out_labels, double *out_scores, size_t *out_counts);
/* nq filtered KNN queries, device pointers end to end, enqueued on `stream` (a cudaStream_t cast to void*, NULL = the legacy
 * default stream); the call returns without waiting for the device.
 * d_queries: nq stored-form query blobs, laid out as for VecSimB200_TopKQueryBatchDevice (cosine normalised, int8 / uint8 cosine
 * with its norm appended).  d_doc_ids[i]: device pointer to query i's ascending filter docIds; d_counts (nullable) [i]: device
 * pointer to its u32 count, read in stream order (NULL, or a NULL entry: caps[i] is the exact count); caps[i]: a host upper bound on
 * that count (II_ResultSet_Capacity of an AND from II_IntersectBatchDevice; 0 = an empty filter, its pointers are not read).  The
 * three pointer arrays are host arrays.
 * Out: [nq][k] int64 labels (-1 = empty) and float distances (NaN = empty), ascending by (distance, docId); d_out_counts (nullable)
 * [nq] u32 entries per query.  Every row is exactly what VecSimB200_TopKFiltered answers for that query and filter: absent or
 * deleted docIds score NaN and are skipped, multi-value indexes take its fold, and distance bits are the same.
 * Single- and multi-value indexes, k <= 1024.  The launches do not depend on nq: one ragged gather over the caps, 2 ceil(k / 128)
 * segmented selects and one unpack (DESIGN.md §4.6).
 * Host waits: none once the index has no pending mutation.  After rows or labels changed, the first call flushes staged rows and
 * rebuilds the docId -> rows table, which waits for those copies; a call needing more scratch than any before it grows the
 * index's device scratch, which waits for the device.  The scratch is shared with VecSimB200_TopKQueryBatchDevice and reused call
 * after call in stream order: enqueue both on one stream (or synchronise between streams), and do not mutate the index while a
 * batch is in flight.
 * Returns 0 (also for nq == 0 or k == 0: nothing is enqueued); -1 for k > 1024 or a CUDA failure; -2, before anything is enqueued,
 * for labels too sparse for the dense table or a cap beyond the 32-bit id range (the same rules as VecSimB200_TopKFiltered). */
int VecSimB200_TopKFilteredBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                       const uint32_t *const *d_counts, const size_t *caps, int64_t *d_out_labels, float *d_out_scores,
                                       uint32_t *d_out_counts, void *stream);
/* The same batch, each query answered by one of two device routes (the device counterpart of hybrid_reader.c's mode choice,
 * DESIGN.md §4.10).  HYBRID_ADHOC_BF: the ragged gather of VecSimB200_TopKFilteredBatchDevice.  HYBRID_BATCHES: the fp32
 * tensor-core route of VecSimB200_TopKQueryBatchDevice (sample pass, fixed-bound main pass, exact rescoring and proof) with the
 * filter applied to the rows, its open queries finished by the gather.  Every row equals, bit for bit, the row
 * VecSimB200_TopKFilteredBatchDevice returns for the same query and filter (labels, distances, counts, exact ties at the k-th
 * place resolved by docId); only the route and its cost differ.  Filter lists must be STRICTLY ascending, as every II_* set is.
 * Arguments, outputs, stream and return codes are those of VecSimB200_TopKFilteredBatchDevice; in addition -1 for a
 * queryParams->searchMode other than EMPTY_MODE (0), HYBRID_ADHOC_BF and HYBRID_BATCHES.  batchSize is not read.
 * queryParams NULL or searchMode 0: each query's route is chosen on the host from its cap, n, dim, k and the queries that would
 * share the dense pass (DESIGN.md §4.10); HYBRID_ADHOC_BF forces the gather, HYBRID_BATCHES the dense route for every query
 * where the batch is eligible: a single-value FLOAT32 index in coarse mode 1 with the fixed bound on (VECSIM_B200_FIXED), dim % 8
 * == 0 in 32..1024, >= 65536 rows within the fp16 range, and 16 dense queries or more unless the fp16 shadow is already built.
 * Elsewhere every query takes the gather.  out_modes (nullable host [nq]): the route of each query, written before the call
 * returns.  After a synchronise, VecSimB200_LastCoarseFlags gives per query 1 / 2 = proven by the first / second tier, 0 =
 * answered by the gather (every ad-hoc query); VecSimB200_LastBatchPath is 1 when any query took the dense route, and the
 * index's last search mode HYBRID_BATCHES then, else HYBRID_ADHOC_BF.
 * Host waits: those of VecSimB200_TopKFilteredBatchDevice, and the first build of the fp16 shadow (or its refresh after
 * mutations).  Launches do not depend on nq: 2 + 2 ceil(k / 128) with no dense query; with dense queries 10 + 2 ceil(k / 128),
 * +1 for L2 / inner product and +4 for the second tier (on unless VECSIM_B200_TIER2=0). */
int VecSimB200_HybridTopKBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                     const uint32_t *const *d_counts, const size_t *caps, VecSimQueryParams *queryParams, int64_t *d_out_labels,
                                     float *d_out_scores, uint32_t *d_out_counts, int *out_modes, void *stream);
/* nq filtered range queries ("@tag:{...} @v:[VECTOR_RANGE $r $B]"), device pointers end to end (DESIGN.md §4.13).  d_queries,
 * d_radii, cap (1..4096), order, the outputs and stream as in VecSimB200_LabelRangeQueryBatchDevice; d_doc_ids, d_counts and caps as
 * in VecSimB200_HybridTopKBatchDevice (host arrays of device pointers, counts read in stream order, caps host upper bounds).  Filter
 * lists must be STRICTLY ascending.
 * Query i's answer is exactly VecSimB200_LabelRangeQueryBatchDevice's answer for (query i, d_radii[i]) restricted to the docIds of
 * filter i: the same labels, score bits, order and cap rule, with d_out_counts[i] the true number of such labels.  A docId is in it
 * iff it is live and one of its rows scores <= d_radii[i] (a float compare: a NaN score never passes, a NaN radius keeps nothing, a
 * negative radius is answered as given); its score is the smallest passing row score.  Absent and deleted docIds contribute nothing.
 * Routes: every query can take the range form of the ragged gather of VecSimB200_TopKFilteredBatchDevice.  A single-value batch
 * that VecSimB200_RangeQueryBatchDevice would send to its fp32 or 8-bit tensor-core route can instead take that route as a whole
 * with the filters applied to the rows; the queries it leaves open go to the gather.  queryParams NULL or searchMode 0: the
 * batch goes dense when the bytes its gathers would read exceed what the dense route reads (DESIGN.md §4.13); HYBRID_ADHOC_BF
 * forces the gather, HYBRID_BATCHES the dense route where the batch is eligible.  fp16 / bf16 and multi-value indexes always take
 * the gather.  out_modes (nullable host [nq]): each query's route, written before the call returns.  After a synchronise,
 * VecSimB200_LastCoarseFlags gives 1 per query a dense route answered and 0 per query the gather answered; VecSimB200_LastBatchPath
 * is 1 (fp32 route), 2 (8-bit route) or 0 (gather only).  The index's last search mode is RANGE_QUERY.
 * Host waits: those of VecSimB200_TopKFilteredBatchDevice and VecSimB200_RangeQueryBatchDevice (flush, docId table rebuild, first
 * fp16 shadow or int32 |row|^2 table).  Launches do not depend on nq: 2 on the gather alone; 8 on the fp32 route (+1 for L2 / inner
 * product), 6 on the 8-bit route (+1 for L2).
 * Returns 0 (with nothing enqueued for nq == 0); -1 for cap == 0 or cap > 4096, an order other than BY_ID / BY_SCORE, a searchMode
 * other than 0 / HYBRID_ADHOC_BF / HYBRID_BATCHES, or a CUDA failure; -2, before anything is enqueued, for labels too sparse for
 * the dense docId table or a cap beyond the 32-bit id range (the rules of VecSimB200_TopKFilteredBatchDevice). */
int VecSimB200_HybridRangeQueryBatchDevice(VecSimIndex *index, const void *d_queries, size_t nq, const float *d_radii, size_t cap,
                                           VecSimQueryReply_Order order, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts,
                                           const size_t *caps, VecSimQueryParams *queryParams, int64_t *d_out_labels, float *d_out_scores,
                                           uint32_t *d_out_counts, int *out_modes, void *stream);
/* Batched fp32 queries (cosine, and in mode 1 also L2 and raw inner product; nq >= 16, k <= 16, dim % 8 == 0,
 * >= 65536 rows) take a wgmma coarse
 * pass + exact rescoring from the fp32 rows + a per-query completeness proof, with the exact scan as
 * on-device fallback (csrc/coarse_tc.cu); results are identical either way.  mode: 0 = exact scans only,
 * 1 = coarse pass over an fp16 shadow copy of the rows (+50% HBM, built lazily by the first eligible
 * batch; once it is complete, single VecSimIndex_TopKQuery calls ride it too), 2 = TF32 coarse pass over the fp32 rows
 * (no extra memory, slower than 1),
 * -1 = environment default (VECSIM_B200_COARSE, 1 unless set). */
void VecSimB200_SetCoarseMode(int mode);
/* Debug: after a VecSimB200_TopKQueryBatchDevice call, per-query flags (1 = answered by the tensor-core path on the first
 * tier's candidate lists, 2 = by the second tier's 128-entry lists, 0 = fell back to the exact scan).  Multi-value
 * index: 1 / 2 / 0 as before for its row stage, with the label check passed; 3 = fewer than k labels among the rows the row
 * stage selected, the label-aware exact scan answered (DESIGN.md §4.4).  Returns -1 if the last batch did not take the coarse
 * path. */
int VecSimB200_LastCoarseFlags(VecSimIndex *index, uint32_t *out_ok, size_t nq);
/* Debug: which route the last top-k query (single or batched) took: 0 = exact CUDA-core scan, 1 = tensor-core coarse pass + exact
 * rescoring + proof (fp32 cosine), 2 = tensor-core direct, k <= 128 (csrc/coarse_tc.cu): fp16 / bf16 corpora, inner
 * product or cosine — the fp32-accumulated products of the stored 16-bit values are the distances; int8 / uint8 corpora,
 * inner product, cosine or L2 — s8 / u8 wgmma integer dot products are exact and the reference's float expression is applied
 * to them (L2: float(|row|^2 + |q|^2 - 2 dot), evaluated in int32 from exact squared norms), bit-exact. */
int VecSimB200_LastBatchPath(VecSimIndex *index);
/* Debug: the operand copy of the fp32 rows the last route 1 query or batch read: 8 = the int8 copy (unit rows: cosine with
 * k <= 128), 16 = the fp16 copy, 0 = none (another route, or TF32 on the fp32 rows). */
int VecSimB200_LastCoarseShadowBits(VecSimIndex *index);
/* Library/ABI version and the SM arch the kernels were compiled for ("sm_90a"). */
const char *VecSimB200_Version(void);

#ifdef __cplusplus
}
#endif
#endif /* VECSIM_B200_H */
