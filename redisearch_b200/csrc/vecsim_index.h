// Host-side FLAT index object behind the VecSim C API: label<->row bookkeeping, preprocessing,
// staging of appended rows, query contexts (stream + scratch), reply objects.  The vectors
// themselves live only in HBM.  Mirrors the host logic of
//   VS/algorithms/brute_force/brute_force.h            (append / swap-delete / queries / heuristics)
//   VS/algorithms/brute_force/brute_force_single.h     (label -> id, update in place)
//   VS/algorithms/brute_force/brute_force_multi.h      (label -> ids)
//   VS/algorithms/brute_force/bf_batch_iterator.h      (batch iterator state machine)
#pragma once
#include "../../include/vecsim_b200.h"
#include "coarse_tc.h"
#include "vecsim_kernels.h"

#include <atomic>
#include <map>
#include <memory>
#include <limits>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

struct VecSimQueryResult {
    size_t id;
    double score;
};
struct VecSimQueryReply {
    std::vector<VecSimQueryResult> results;
    VecSimQueryReply_Code code = VecSim_QueryReply_OK;
};
struct VecSimQueryReply_Iterator {
    VecSimQueryReply *reply;
    size_t pos;
};
struct VecSimDebugInfoIterator {
    std::vector<VecSim_InfoField> fields;
    std::vector<std::string> owned;
    size_t pos = 0;
};

namespace rsb200 {

class BatchScratch;

struct Globals {
    std::atomic<timeoutCallbackFunction> timeout_cb{nullptr};
    std::atomic<logCallbackFunction> log_cb{nullptr};
    VecSimMemoryFunctions mem{};
    std::mutex test_ctx_mu; // VecSim_SetTestLogContext
    std::string test_name, test_type;
};
Globals &globals();
void set_coarse_mode(int mode); // -1 env default, 0 exact scans only, 1 coarse pass on fp16 shadow rows, 2 TF32 coarse pass

// Device + pinned scratch for one in-flight query (or query batch).  Checked out of a pool so
// that many RediSearch worker threads can query one index concurrently (SURVEY.md §8b threading).
struct QueryCtx {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    uint8_t *d_query = nullptr, *h_query = nullptr; // staged query blobs
    size_t query_cap = 0;
    uint64_t *d_cand = nullptr;
    size_t cand_cap = 0;
    uint64_t *d_out = nullptr, *h_out = nullptr;
    size_t out_cap = 0;
    float *d_scores = nullptr; // unfused path: one score per row
    size_t scores_cap = 0;
    uint32_t *d_count = nullptr, *h_count = nullptr;
    uint32_t *d_last_ok = nullptr; // coarse path: per-query verification flags of the last batch (inside d_cand)
    uint32_t last_ok_n = 0;
    uint32_t *d_ids = nullptr, *h_ids = nullptr;
    float *d_dist = nullptr, *h_dist = nullptr;
    size_t ids_cap = 0;
    uint64_t *d_lab = nullptr; // label stage of a multi-value batch (its flags stay readable after the call)
    size_t lab_cap = 0;
    bool abandoned = false; // a timed-out caller left while kernels were still running on `stream`: synchronise before reuse
    // raised by the host when a caller times out: the exact-scan kernel polls it (mapped pinned memory) and winds down, so the GPU
    // does not finish a pass nobody waits for
    uint32_t *h_abort = nullptr;
    const uint32_t *d_abort = nullptr;
    ~QueryCtx();
    bool init();
    bool need_query(size_t bytes);
    bool need_cand(size_t elems);
    bool need_out(size_t elems);
    bool need_scores(size_t n);
    bool need_ids(size_t n);
    bool need_lab(size_t elems);

  private:
    // once the stream is idle: frees d (and its pinned mirror *h), then allocates new_cap elements for each; cap = new_cap on success
    template <class T> bool grow(T *&d, size_t &cap, size_t new_cap, T **h = nullptr);
};

class FlatIndex;

struct BatchIter {
    FlatIndex *index;
    std::vector<uint8_t> query; // stored-form query blob (normalised for cosine)
    void *timeout_ctx;
    std::unique_ptr<QueryCtx> ctx; // owns the score array between Next calls
    bool scored = false;
    uint32_t n_rows = 0;        // rows at scoring time
    size_t label_count = 0;     // labels at scoring time (bf_batch_iterator.h:29)
    size_t returned = 0;
    bool has_cursor = false;
    uint64_t cursor = 0;                  // last composite handed out
    std::unordered_set<size_t> seen;      // multi-value: labels already returned
    std::vector<size_t> id_to_label_snap; // label table at scoring time
};

struct AdhocCtx {
    FlatIndex *index;
    std::vector<uint8_t> query; // stored-form query
    std::unique_ptr<QueryCtx> ctx;
    bool query_on_device = false;
};

class FlatIndex {
  public:
    static FlatIndex *create(const BFParams &p, void *log_ctx);
    ~FlatIndex();

    int add(const void *blob, size_t label);
    int add_bulk(const void *blobs, size_t stride, size_t n, const size_t *labels, size_t label0);
    int add_bulk_device(const void *d_rows, size_t n, size_t label0);
    int remove(size_t label);
    size_t size() const { return count_; }
    size_t label_count() const { return multi_ ? label_to_ids_.size() : label_to_id_.size(); }
    bool reserve(size_t rows);
    bool flush();

    VecSimQueryReply *topk(const void *q, size_t k, VecSimQueryParams *qp, VecSimQueryReply_Order order);
    // the same through the request combiner (micro_batcher.h): concurrent callers share one corpus pass.  Opt-in:
    // VECSIM_B200_MICROBATCH_US=<collection window in microseconds> (default 0 = off).
    VecSimQueryReply *topk_combined(const void *q, size_t k, VecSimQueryParams *qp, VecSimQueryReply_Order order);
    static int microbatch_window_us();
    int topk_batch(const void *qs, size_t qstride, size_t nq, size_t k, VecSimQueryParams *qp, size_t *out_labels,
                   double *out_scores);
    int topk_batch_device(const void *d_q, size_t nq, size_t k, int64_t *d_labels, float *d_scores, cudaStream_t s);
    VecSimQueryReply *range(const void *q, double radius, VecSimQueryParams *qp, VecSimQueryReply_Order order);
    // nq range queries, replies[i] = what range(qs + i * qstride, radii[i], qp, order) returns.  Eligible fp32 batches take
    // the fixed-bound tensor-core pass + exact rescoring + proof (DESIGN.md §4); out_flags[i] (nullable) = 1 for a query
    // answered there, 0 for one answered by range().  Arguments are validated by the caller.
    int range_batch(const void *qs, size_t qstride, size_t nq, const double *radii, VecSimQueryParams *qp, VecSimQueryReply_Order order,
                    VecSimQueryReply **replies, uint32_t *out_flags);
    // the same with device pointers end to end, stream-ordered: VecSimB200_RangeQueryBatchDevice (DESIGN.md §4.11)
    int range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_labels,
                           float *d_scores, uint32_t *d_counts, cudaStream_t s);
    // the same answered per label on any index: VecSimB200_LabelRangeQueryBatchDevice (DESIGN.md §4.12)
    int label_range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_labels,
                                 float *d_scores, uint32_t *d_counts, cudaStream_t s);
    // the same restricted to a filter per query, on the ragged gather or a filtered tensor-core route:
    // VecSimB200_HybridRangeQueryBatchDevice (DESIGN.md §4.13)
    int hybrid_range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order,
                                  const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps, VecSimQueryParams *qp,
                                  int64_t *d_labels, float *d_scores, uint32_t *d_counts_out, int *out_modes, cudaStream_t s);
    double distance_from(size_t label, const void *stored_form_blob);
    bool prefer_adhoc(size_t subset, size_t k, bool initial);

    BatchIter *batch_new(const void *q, VecSimQueryParams *qp);
    VecSimQueryReply *batch_next(BatchIter *it, size_t n, VecSimQueryReply_Order order);

    AdhocCtx *adhoc_new(const void *q);
    void adhoc_distances(AdhocCtx *c, const size_t *labels, double *out, size_t n);
    // fused hybrid ad-hoc query: k nearest among the rows whose labels are listed (ascending) in doc_ids
    int topk_filtered(const void *q, size_t k, const uint32_t *doc_ids, size_t n, bool ids_on_device, size_t *out_labels,
                      double *out_scores, size_t *out_count);
    int topk_filtered_batch(const void *const *queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids, const size_t *counts,
                            size_t *out_labels, double *out_scores, size_t *out_counts);
    // the same, device pointers end to end and stream-ordered: VecSimB200_TopKFilteredBatchDevice
    int topk_filtered_batch_device(const void *d_q, size_t nq, size_t k, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts,
                                   const size_t *caps, int64_t *d_labels, float *d_scores, uint32_t *d_counts_out, cudaStream_t s);
    // the same rows, each query on the ragged gather or on the filtered tensor-core route: VecSimB200_HybridTopKBatchDevice
    int hybrid_topk_batch_device(const void *d_q, size_t nq, size_t k, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts,
                                 const size_t *caps, VecSimQueryParams *qp, int64_t *d_labels, float *d_scores, uint32_t *d_counts_out,
                                 int *out_modes, cudaStream_t s);

    VecSimIndexBasicInfo basic_info() const;
    VecSimIndexStatsInfo stats_info() const;
    VecSimIndexDebugInfo debug_info() const; // BruteForceIndex::debugInfo, brute_force.h:318-325
    VecSimDebugInfoIterator *debug_iterator() const;
    void set_last_mode(VecSearchMode m) { last_mode_ = m; }
    VecSimB200_Stats get_stats(bool reset);
    // debug: verification flags of the last device-batch call (1 = answered by the tensor-core path)
    int last_coarse_flags(uint32_t *out, size_t n);
    const void *device_rows(size_t *pitch, size_t *rows) {
        flush();
        *pitch = pitch_;
        *rows = count_;
        return d_rows_;
    }

    // stored-form rows [first, first + n) -> tightly packed host buffer (stored_bytes_ per row); false if out of range
    bool read_rows(size_t first, size_t n, void *host_dst);
    size_t query_blob_bytes() const { return stored_bytes_; } // VecSimParams_GetQueryBlobSize
    void preprocess_query(const void *blob, uint8_t *dst) const;   // -> stored form
    void preprocess_storage(const void *blob, uint8_t *dst) const; // -> stored form

    VecSimType type_;
    VecSimMetric metric_;
    size_t dim_;
    bool multi_;
    size_t block_size_;
    void *log_ctx_;

    void log(const char *level, const char *fmt, ...) const;

  private:
    FlatIndex() = default;
    CorpusView view() const;
    std::unique_ptr<QueryCtx> checkout();
    void checkin(std::unique_ptr<QueryCtx> c);
    bool grow_to(size_t rows);
    bool sync_labels_to_device();
    bool timed_out(void *ctx) const;
    // Wait for `s`, polling the timeout callback (VecSim_SetTimeoutCallbackFunction) every ~50 us while kernels run —
    // the reference checks it per vector (brute_force.h:265-269); a device pass cannot be interrupted, but the caller
    // is released as soon as the deadline passes.  0 = done, 1 = timed out (the stream is still busy), -1 = CUDA error.
    int wait_polling(cudaStream_t s, void *timeout_ctx) const;
    // wait_polling on c's stream; on a timeout c is marked abandoned and its running kernels are told to wind down (h_abort)
    int wait_or_abandon(QueryCtx &c, void *timeout_ctx) const;
    // a scan over `bytes` of rows into the stats, timed by c's events (c == NULL: untimed)
    void record_scan(const QueryCtx *c, uint64_t bytes);
    // k smallest composites (> cursor) over ctx->d_scores[0..n) into ctx->h_out, chunked by
    // kMaxFusedK; returns the number found or -1.
    long select_from_scores(QueryCtx &c, uint32_t n, bool has_cursor, uint64_t cursor, size_t want);
    size_t query_pitch() const { return (stored_bytes_ + 15) & ~(size_t)15; } // bytes between staged queries
    size_t f16_query_pitch() const { return (dim_ * 2 + 15) & ~(size_t)15; } // bytes between the fp16 forms of fp32 queries
    // nq query blobs, `stride` bytes apart -> c.d_query, query_pitch() apart and zero-padded, then `tail_bytes` of `tail`.  raw:
    // the blobs are put in stored form (preprocess_query); else they are in stored form already
    bool stage_queries(QueryCtx &c, const void *blobs, size_t stride, size_t nq, bool raw, const void *tail = nullptr, size_t tail_bytes = 0);
    // [nq][ke] best composites of a batch: rows of a single-value index, labels (score, best row) of a multi-value one
    bool batch_scan(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t ke, cudaStream_t st, LaunchCounters &lc,
                    uint64_t **d_result);
    // row-level routes; tc_only: only a tensor-core route runs, else nothing is launched and *d_result = NULL
    bool batch_scan_rows(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t ke, cudaStream_t st, LaunchCounters &lc,
                         uint64_t **d_result, bool tc_only = false);
    // multi-value index: the first kl distinct labels per query (DESIGN.md §4.4); needs d_id_to_label_ in sync
    bool batch_scan_labels(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t kl, cudaStream_t st, LaunchCounters &lc,
                           uint64_t **d_result, bool host_fallback = false);

    // fp32 queries -> the operands of a pass over the fp16 shadow: their fp16 form in q16 (f16_query_pitch() apart) and, where d_qn2
    // is not NULL (rows not all unit), |q|^2 in d_qn2
    bool shadow_operands(const void *d_q, size_t qpitch, uint32_t nq, uint8_t *q16, float *d_qn2, cudaStream_t st, LaunchCounters &lc,
                         CoarseOperands &ops);
    // the operands of a pass over 8-bit rows; int8 / uint8 L2: the exact int32 |q|^2 into d_qn and the |row|^2 table (ensure_shadow)
    bool direct8_operands(const void *d_q, size_t qpitch, uint32_t nq, int32_t *d_qn, cudaStream_t st, LaunchCounters &lc, CoarseOperands &ops);
    // false when the fp32 rows hold values outside the fp16 range (or NaN): the index stays on the exact scans from now on
    bool shadow_values_in_range();

    // The fixed-bound range route (DESIGN.md §4.11) of one batch, over the fp16 shadow (CoarseF16), the stored 16-bit rows
    // (CoarseDirect16) or the 8-bit rows (CoarseDirect8).  Its scratch is carved from the caller's batch layout by take().
    struct RangeScratch {
        uint64_t *cand = nullptr, *list_scratch = nullptr;
        uint8_t *q16 = nullptr;
        float *qn2 = nullptr, *thr = nullptr;
        uint32_t *ovf = nullptr, *front = nullptr;
        void take(BatchScratch &s, const FlatIndex &ix, CoarseKind kind, const CoarsePlan &cp, uint32_t nq, bool fold);
    };
    // Where the route writes its answers.  flags == NULL: the proven hits of query q, rows as (score key, row) composites, go to
    // hits[q * cap, ...) with cnt[q] = their number (cap != 0), or packed at hits[off[q], ...) with *total = their sum (cap == 0;
    // CoarseF16 only); ok[q] = 1 for a proven query.  flags != NULL (multi-value index): the label fold of launch_range_label_fold
    // into hits[q * cap, ...), with LastCoarseFlags in flags.
    struct RangeOut {
        uint64_t *hits;
        uint32_t cap;
        uint32_t *ok, *cnt, *off, *total, *flags;
    };
    // the route's query operands, bound, main pass (timed by c's events) and rescoring or packing; bm / words (nullable): filter
    // bitmaps of the batch's queries
    bool enqueue_range_route(QueryCtx &c, const CorpusView &v, CoarseKind kind, const CoarsePlan &cp, const RangeScratch &r, const void *d_q,
                             size_t qpitch, uint32_t nq, const float *d_radii, const uint32_t *bm, uint32_t words, const RangeOut &out,
                             cudaStream_t st, LaunchCounters &lc);

    // The plans of the shadow KNN tier chain (DESIGN.md §4.2, §4.5): the main pass (a fixed-bound pass after a sample pass when
    // two_pass, else adaptive lists) and the second tier for the queries the first proof left open.
    struct KnnTiers {
        CoarsePlan main{}, sample{}, second{};
        bool two_pass = false, tier2 = false;
    };
    // aim / tiles_per_k: the sample pass's stride (sample_stride); filt: the main pass runs with row filters
    static KnnTiers plan_knn_tiers(const CorpusView &v, uint32_t nq, CoarseKind kind, uint32_t ke, double aim, double tiles_per_k, bool filt);
    struct KnnScratch {
        uint64_t *cand = nullptr, *cand_s = nullptr, *cand_t2 = nullptr, *list_scratch = nullptr;
        uint8_t *q = nullptr, *q_t2 = nullptr; // the queries in the operand type of the copy, and tier 2's open ones
        float *qn2 = nullptr, *qn2_t2 = nullptr, *qeps = nullptr, *qeps_t2 = nullptr, *thr = nullptr;
        uint32_t *ok = nullptr, *idx = nullptr, *n2 = nullptr, *ovf = nullptr;
        uint32_t *cnt = nullptr; // [nq][main.grid_x] entries per list of the int8 copy's fixed pass (NULL on the other routes)
        // q_pitch: bytes per operand query row; norms: |q|^2 per query (rows not all unit); q8: the int8 copy's eps per query
        void take(BatchScratch &s, const KnnTiers &t, uint32_t nq, size_t q_pitch, bool norms, bool q8);
    };
    // sample pass, bound, main pass (timed by c's events), exact rescoring + proof into out [nq][ke] and ok, then the second tier.
    // ops: the first tier's operands over the copy (their queries and |q|^2 in s); d_q32: the fp32 queries the rescoring reads.
    // bm / words / row_label (nullable): filter bitmaps of the queries and the docId of each row (answers carry it, ties resolve by it)
    bool enqueue_knn_tiers(QueryCtx &c, const CorpusView &v, CoarseKind kind, const KnnTiers &t, const KnnScratch &s, const CoarseOperands &ops,
                           const void *d_q32, size_t qpitch, uint32_t nq, uint32_t ke, uint64_t *out, const uint32_t *bm, uint32_t words,
                           const uint64_t *row_label, cudaStream_t st, LaunchCounters &lc);

    // [docId pointers nq][count pointers nq][score offsets nq + 1][first chunks nq + 1], then the caller's u32 words `tail`: filled in a
    // pinned table slot and uploaded to d_tab (ragged_table_elems(nq, tail.size()) words) on st.  False when no slot can be had;
    // ok &= the upload was enqueued
    static size_t ragged_table_elems(size_t nq, size_t tail_words) { return 4 * nq + 2 + (tail_words + 1) / 2; }
    bool upload_ragged_table(uint64_t *d_tab, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps, uint32_t nq,
                             const std::vector<uint32_t> &tail, cudaStream_t st, RaggedBatch &b, bool &ok);
    void finish_reply(VecSimQueryReply *rep, VecSimQueryReply_Order order) const;

    DType dtype_;
    MetricKind mkind_;
    size_t elem_bytes_ = 0;   // sizeof element
    size_t stored_bytes_ = 0; // VS/utils/vec_utils.cpp:296-302
    size_t pitch_ = 0;        // HBM row pitch (>= stored_bytes_)

    uint8_t *d_rows_ = nullptr;
    // fp16 copy of the fp32 rows for the tensor-core coarse pass, stored tile by tile in the swizzled layout
    // the kernel streams (coarse_tc.cu); built lazily by the first eligible batch, rows [0, shadow_rows_)
    // valid except shadow_dirty_
    uint8_t *d_shadow_ = nullptr;
    size_t shadow_cap_ = 0, shadow_rows_ = 0;
    // int8 copy of unit rows for the cosine batches with k <= kCoarseMaxK (DESIGN.md §4.2), the same tiled layout with one byte per
    // element and one scale per 128-row tile (d_tscale_); built lazily by the first batch that takes it and kept by the same
    // bookkeeping as the fp16 copy.  d_stats8_ = running maxima (float bits) of the quantization residual norm and of the row norm
    // over every row quantized since the last full rebuild, mirrored on the host after each refresh
    uint8_t *d_shadow8_ = nullptr;
    float *d_tscale_ = nullptr;
    uint32_t *d_stats8_ = nullptr;
    float shadow8_delta_ = 0.0f, shadow8_xmax_ = 0.0f;
    // L2 / raw inner-product indexes: |row|^2 per row and the running maxima the error bound needs.  int8 / uint8 L2 indexes keep
    // the exact int32 |row|^2 here (stored as int32, no shadow, no maxima) for the integer tensor-core route; fp16 / bf16 indexes
    // keep |row|^2 of their stored rows and its running maximum (no shadow) once a range batch takes the direct 16-bit route.
    // The same shadow_rows_ / shadow_dirty_ / shadow_cap_ bookkeeping tracks it
    float *d_norm2_ = nullptr;
    uint32_t *d_stats_ = nullptr;
    float shadow_max_norm_ = 0.0f, shadow_max_abs_ = std::numeric_limits<float>::infinity();
    std::atomic<bool> coarse_disabled_{false}; // L2 / IP index with values outside the fp16 range: exact scans only
    // cosine index that took an in-place update (brute_force_single.h:139-144 stores the caller's RAW blob): its rows are
    // no longer all unit vectors, the coarse proof uses the norm-scaled bound from then on
    std::atomic<bool> raw_rows_{false};
    bool unit_rows() const { return metric_ == VecSimMetric_Cosine && !raw_rows_; }
    std::vector<idType> shadow_dirty_;
    // a per-row copy (the fp16 shadow and / or |row|^2) exists: in-place overwrites and swap-deletes go to shadow_dirty_
    bool keeps_row_copies() const { return d_shadow_ || d_shadow8_ || d_norm2_; }
    bool int_l2() const { return (dtype_ == DT_I8 || dtype_ == DT_U8) && mkind_ == MT_L2; }
    // fp32: the fp16 shadow (+ |row|^2 unless unit rows); int8 / uint8 L2: only the int32 |row|^2 table; fp16 / bf16: only |row|^2
    // q8: the int8 copy instead (unit rows); every copy the index already keeps is brought up to date either way
    bool ensure_shadow(cudaStream_t st, bool q8 = false);
    // a KNN batch of this k on this single-value index of unit rows runs on the int8 copy (its bounds are finite once built)
    bool q8_route(uint32_t nq, uint32_t ke) const;
    void disable_coarse(); // rows outside the fp16 range: exact scans from now on, the shadow's HBM is given back
    bool single_query_takes_coarse(uint32_t ke, const float *host_query = nullptr, bool q8 = false);
    size_t capacity_ = 0; // rows of HBM allocated
    size_t count_ = 0;    // rows in the index (incl. staged)
    size_t resident_ = 0; // rows already copied to HBM
    uint8_t *h_stage_ = nullptr; // pinned; rows [resident_, count_)
    size_t stage_cap_rows_ = 0;
    cudaStream_t copy_stream_ = nullptr;

    std::vector<size_t> id_to_label_;
    std::unordered_map<size_t, idType> label_to_id_;
    std::unordered_map<size_t, std::vector<idType>> label_to_ids_;
    // multi-value index: rows per label -> number of labels with that many rows; its largest key is m, the most rows any label
    // owns, which sizes the row stage of a batch (DESIGN.md §4.4)
    std::map<size_t, size_t> rows_per_label_;
    void label_rows_changed(size_t from, size_t to); // a label went from `from` to `to` rows (0 = absent); caller holds mu_
    size_t max_rows_per_label() const;
    uint64_t *d_id_to_label_ = nullptr;
    size_t d_labels_cap_ = 0;
    bool labels_dirty_ = true;
    // dense label -> row id table on the device (labels are RediSearch docIds: small integers), for topk_filtered.  A multi-value
    // index keeps a CSR table instead: d_label_to_id_ holds offsets [l2i_size_ + 1], d_label_rows_ the rows [count_] of each label
    // in label_to_ids_ order (the order the reference's min fold visits them).  l2i_size_ = largest label + 1.
    uint32_t *d_label_to_id_ = nullptr;
    size_t l2i_size_ = 0, l2i_cap_ = 0;
    uint32_t *d_label_rows_ = nullptr;
    size_t label_rows_cap_ = 0;
    bool l2i_dirty_ = true;
    bool sync_label_table();
    // the body of range_batch_device / label_range_batch_device: per row on a single-value index, per label on a multi-value one
    int range_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_labels,
                     float *d_scores, uint32_t *d_counts, cudaStream_t s);

    mutable std::mutex mu_;      // guards mutation + staging
    std::mutex pool_mu_;
    std::vector<std::unique_ptr<QueryCtx>> pool_;
    mutable VecSearchMode last_mode_ = EMPTY_MODE;

    std::atomic<uint64_t> launches_total_{0};
    std::atomic<uint64_t> coarse_batches_{0};
    bool last_batch_coarse_ = false;
    int last_batch_path_ = 0; // 0 exact scan, 1 tensor-core coarse pass + proof, 2 tensor-core direct (16-bit corpora); multi-value: the row stage's
  public:
    int last_batch_path() const { return last_batch_path_; }
    int last_shadow_bits_ = 0; // the copy route 1 read: 8 int8, 16 fp16, 0 none
    int last_shadow_bits() const { return last_shadow_bits_; }
  private:
    std::unique_ptr<QueryCtx> dev_ctx_; // scratch of topk_batch_device / topk_filtered_batch_device (stream-ordered)
    std::mutex dev_mu_;
    // pinned staging of topk_filtered_batch_device's pointer tables (under dev_mu_): a slot is reused once the event recorded after
    // its upload has completed; while every slot is still in flight a new one is added, so the host never waits for the upload
    struct TableSlot {
        uint64_t *h = nullptr;
        size_t cap = 0; // uint64 elements
        cudaEvent_t ev = nullptr;
    };
    std::vector<TableSlot> table_ring_;
    TableSlot *table_slot(size_t elems);
    bool dev_timing_pending_ = false;
    uint64_t dev_timing_bytes_ = 0;
    void collect_dev_timing_locked();
    std::atomic<uint64_t> scan_launches_{0};
    std::atomic<uint64_t> scan_bytes_{0};
    double scan_us_ = 0;
    std::mutex stats_mu_;
    struct TopkReq;
    std::mutex mb_mu_;
    std::map<size_t, std::shared_ptr<void>> batchers_; // one MicroBatcher<TopkReq> per k
    friend struct BatchIter;
};

} // namespace rsb200
