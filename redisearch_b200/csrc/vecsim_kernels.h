// Host-visible launchers of the sm_90a KNN kernels (vecsim_kernels.cu).  Plain CUDA runtime
// types only; no torch.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace rsb200 {

enum DType : int { DT_F32 = 0, DT_F16 = 1, DT_BF16 = 2, DT_I8 = 3, DT_U8 = 4 };
// MT_COS only differs from MT_IP for the integer types (division by the stored norms,
// VS/spaces/IP/IP.cpp:264-285); float corpora are normalised at ingest and use IP arithmetic
// (VS/spaces/spaces.cpp:50-61).
enum MetricKind : int { MT_L2 = 0, MT_IP = 1, MT_COS = 2 };

struct CorpusView {
    const void *rows;   // device, row-major, `pitch` bytes per row
    size_t pitch;       // >= stored row size, multiple of 16 for the 16/8-bit types
    uint32_t n_rows;
    uint32_t dim;
    DType dtype;
    MetricKind metric;
};

struct LaunchCounters {
    uint64_t launches = 0;
};

int device_sm_count();

// ---- fused scan + per-warp top-k (k <= kMaxFusedK) -------------------------------------------
// Shape of the candidate buffer the scan writes: lists_per_query lists of k composites per query.
struct ScanPlan {
    uint32_t grid_x, grid_y, wq, qt, lists_per_query;
    size_t smem_bytes;
    size_t cand_elems; // uint64 elements needed in d_cand
    bool labels;       // label-aware lists (multi-value index)
    bool q_smem;       // the queries are staged in shared memory
};
// labels: plan the label-aware variant (lists of distinct labels, a label per slot in shared memory)
ScanPlan plan_scan_topk(const CorpusView &c, uint32_t nq, uint32_t k, bool labels = false);
// d_queries: nq device blobs, qpitch bytes apart, already in stored form (normalised etc.).
// d_id_to_label (label-aware plans only, else NULL): row -> label; each list then holds the k best distinct labels it has seen,
// each at its best (score, row) composite (DESIGN.md §4.4), to be reduced with launch_final_select_labels.
cudaError_t launch_scan_topk(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq,
                             uint32_t k, const ScanPlan &plan, uint64_t *d_cand, cudaStream_t s,
                             LaunchCounters *ctr, const uint32_t *d_q_ok = nullptr, const uint32_t *d_abort = nullptr,
                             const uint64_t *d_id_to_label = nullptr);
// label-aware lists -> per query the first k distinct labels of the sorted union, as (score, best row) composites, ascending,
// kEmptySlot-padded
cudaError_t launch_final_select_labels(const uint64_t *d_cand, uint32_t nq, uint32_t m_per_query, uint32_t k, const uint64_t *d_id_to_label,
                                       uint64_t *d_out, cudaStream_t s, LaunchCounters *ctr);
// Label stage after a row-level route: d_rows [nq][K] ascending composites -> d_out [nq][kl], the first kl distinct labels.
// d_lab_ok[q] = 1 iff the K rows hold at least kl distinct labels (the selection is then exact); d_flags[q] = d_row_ok[q] (1 if
// d_row_ok is NULL) when it holds, else 3.
cudaError_t launch_label_select(const uint64_t *d_rows, uint32_t nq, uint32_t K, const uint64_t *d_id_to_label, uint32_t kl,
                                const uint32_t *d_row_ok, uint64_t *d_out, uint32_t *d_lab_ok, uint32_t *d_flags, cudaStream_t s,
                                LaunchCounters *ctr);
// out[q] = ok[q] ? a[q] : b[q] for [nq][k] composite arrays
cudaError_t launch_blend(const uint32_t *d_ok, const uint64_t *d_a, const uint64_t *d_b, uint32_t nq, uint32_t k, uint64_t *d_out,
                         cudaStream_t s, LaunchCounters *ctr);
// Reduce m_per_query candidate composites per query to the k smallest, ascending.
// d_out: [nq][k] composites (kEmptySlot-padded when fewer than k real candidates exist).
// d_nq_dev (nullable): only the first *d_nq_dev queries are processed (count known on the device only).
cudaError_t launch_final_select(const uint64_t *d_cand, uint32_t nq, uint32_t m_per_query, uint32_t k,
                                uint64_t *d_out, cudaStream_t s, LaunchCounters *ctr, const uint32_t *d_nq_dev = nullptr);

// ---- unfused path: all distances of one query, then cursor-select / range-compact ------------
cudaError_t launch_scan_scores(const CorpusView &c, const void *d_query, float *d_scores,
                               cudaStream_t s, LaunchCounters *ctr);
// k (<= kMaxFusedK) smallest composites strictly greater than *d_cursor (d_cursor may be NULL =
// no lower bound) among scores[0..n).  Writes lists to d_cand (size from plan_select_scores), to
// be reduced with launch_final_select.
uint32_t plan_select_scores_lists(uint32_t n);
cudaError_t launch_select_scores(const float *d_scores, uint32_t n, const uint64_t *d_cursor, uint32_t k,
                                 uint64_t *d_cand, cudaStream_t s, LaunchCounters *ctr);

// ---- exact top-k of a batch for kMaxFusedK < k <= kMaxWideK (DESIGN.md §4.5) --------------------
// The unfused path of one query with a query dimension: per group of `group` batch positions one scan of all their scores
// (score_elems floats of HBM) and ceil(k / 128) cursor selects of up to 128 (cand_elems uint64 of lists).
struct WidePlan {
    uint32_t group, sel_grid;
    size_t score_elems, cand_elems;
};
WidePlan plan_topk_wide(uint32_t n_rows, uint32_t nq);
// Batch positions p < *d_count (nq when d_count is NULL; read on the device) get the exact answer of query d_pos[p] (p when
// d_pos is NULL) in d_out[query][0, k), ascending composites, as the single-query path computes them.  Rows of other queries are
// left alone.  1 + 2 ceil(k / 128) launches per group; a launch whose positions are all dead exits at once.  k <= n_rows.
cudaError_t launch_topk_wide(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t k, const uint32_t *d_pos,
                             const uint32_t *d_count, const WidePlan &p, float *d_scores, uint64_t *d_cand, uint64_t *d_out,
                             const uint32_t *d_abort, cudaStream_t s, LaunchCounters *ctr);
// ---- device range batches (DESIGN.md §4.11) --------------------------------------------------------
constexpr uint32_t kRangeDeviceMaxCap = 4096; // largest per-query result capacity (range_finish_kernel sorts in shared memory)
// The exact range answer of the queries at batch positions p < *d_count (nq without d_count) — query d_pos[p] (p without
// d_pos) — by the scores of launch_topk_wide's grouping (the single-query range() bits): composites of the rows with
// score <= d_radii[q] into d_out[q * cap, ...) unordered, atomically counted in d_counts[q] (zeroed by the caller), past cap
// too.  2 launches per group; a launch whose positions are all answered exits at once.  label_off != NULL (multi-value index,
// DESIGN.md §4.12): the answer is per label instead — label_off [n_labels + 1] / label_rows the CSR label -> rows table, and each
// label with a passing row contributes one composite, its smallest (score key, row), counted per label.
cudaError_t launch_range_wide(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, const uint32_t *d_pos,
                              const uint32_t *d_count, const WidePlan &p, float *d_scores, const float *d_radii, uint32_t cap, uint64_t *d_out,
                              uint32_t *d_counts, const uint32_t *d_abort, cudaStream_t s, LaunchCounters *ctr, const uint32_t *label_off = nullptr,
                              const uint32_t *label_rows = nullptr, uint32_t n_labels = 0);
// Row q of d_labels [nq][cap] holds d_counts[q] composites (as uint64): they become labels (int64) and scores in reply order,
// BY_SCORE (score, label) or BY_ID (label), padded with -1 / NaN; a count past cap pads the whole row.  One launch.
cudaError_t launch_range_finish(int64_t *d_labels, float *d_scores, const uint32_t *d_counts, uint32_t nq, uint32_t cap,
                                const uint64_t *d_id_to_label, bool by_id, cudaStream_t s, LaunchCounters *ctr);
// Append composite(score,id) of every score <= radius to d_out (capacity n), count in *d_count.
cudaError_t launch_range_compact(const float *d_scores, uint32_t n, float radius, uint64_t *d_out,
                                 uint32_t *d_count, cudaStream_t s, LaunchCounters *ctr);

// ---- ad-hoc: distances of listed rows ----------------------------------------------------------
// d_ids[i] == 0xFFFFFFFF -> NaN.
cudaError_t launch_gather_distances(const CorpusView &c, const void *d_query, const uint32_t *d_ids,
                                    uint32_t count, float *d_out, cudaStream_t s, LaunchCounters *ctr);
// Multi-value index: d_out[i] = the reference's min fold (brute_force_multi.h:224-241) over the rows of label d_labels[i],
// label_rows[offsets[l], offsets[l + 1]) in insertion order (CSR, offsets has n_labels + 1 entries); NaN for an absent label.
cudaError_t launch_gather_min_distances(const CorpusView &c, const void *d_query, const uint32_t *d_labels, uint32_t count,
                                        const uint32_t *d_offsets, uint32_t n_labels, const uint32_t *d_label_rows, float *d_out,
                                        cudaStream_t s, LaunchCounters *ctr);

// ---- batched filtered KNN: ragged filter lists whose lengths are known only on the device (DESIGN.md §4.6) ----------------------
// The tables live in device memory.  Query q's scores are scores[off[q], off[q + 1]) (off = prefix sums of the host caps); only the
// first min(*counts[q], cap) entries are live (the whole cap when counts[q] is NULL).
struct RaggedBatch {
    const uint32_t *const *doc_ids; // [nq] query q's ascending docIds
    const uint32_t *const *counts;  // [nq] query q's u32 count, or NULL
    const uint64_t *off;            // [nq + 1]
    uint32_t nq;
};
constexpr uint32_t kRaggedPerBlock = 128; // filter entries per gather CTA
inline uint64_t ragged_blocks(size_t cap) { return (cap + kRaggedPerBlock - 1) / kRaggedPerBlock; }
// distances of every live entry: one launch of n_blocks CTAs, d_blk [nq + 1] = prefix of ragged_blocks over the caps.  Single-value
// index (d_label_rows NULL): d_table maps docId -> row as launch_map_labels; multi-value: CSR offsets over d_label_rows and the fold
// of launch_gather_min_distances.  d_queries: nq stored-form blobs qpitch bytes apart.  max_grid != 0: at most that many CTAs stride
// over the n_blocks chunks (a batch whose counts are mostly 0 does not pay a CTA per chunk of its caps)
cudaError_t launch_gather_ragged(const CorpusView &c, const void *d_queries, size_t qpitch, const RaggedBatch &b, const uint64_t *d_blk,
                                 uint64_t n_blocks, const uint32_t *d_table, uint32_t table_size, const uint32_t *d_label_rows, float *d_scores,
                                 cudaStream_t s, LaunchCounters *ctr, uint64_t max_grid = 0);
// range form (DESIGN.md §4.13): no scores; every live entry whose distance is <= d_radii[q] (a float compare, NaN never passes)
// appends one composite (score key, row) to d_out[q * cap, ...) unordered, atomically counted in d_counts[q] (zeroed by the caller)
// past cap too.  Multi-value: an entry passes iff one of its label's rows does, with the smallest passing (score key, row).  One
// launch, the grid of launch_gather_ragged
cudaError_t launch_gather_ragged_range(const CorpusView &c, const void *d_queries, size_t qpitch, const RaggedBatch &b, const uint64_t *d_blk,
                                       uint64_t n_blocks, const uint32_t *d_table, uint32_t table_size, const uint32_t *d_label_rows,
                                       const float *d_radii, uint32_t cap, uint64_t *d_out, uint32_t *d_counts, cudaStream_t s, LaunchCounters *ctr,
                                       uint64_t max_grid = 0);
// CTAs per query of the segmented select (their lists: parts * 8 per query and chunk)
uint32_t plan_ragged_select_parts(size_t max_cap, uint32_t nq);
// d_out [nq][k] = each query's k smallest (score, position) composites over its live scores, ascending, kEmptySlot-padded;
// k <= kMaxWideK in cursor chunks of kMaxFusedK: 2 ceil(k / 128) launches.  d_cand: nq * parts * 8 * min(k, 128) elements.
cudaError_t launch_topk_ragged(const RaggedBatch &b, const float *d_scores, uint32_t k, uint32_t parts, uint64_t *d_cand, uint64_t *d_out,
                               cudaStream_t s, LaunchCounters *ctr);
// Answer rows of a hybrid batch's tensor-core route (DESIGN.md §4.10): query q with ok[q] != 0 takes row pos[q] of comp [.][k],
// composites (distance, docId).  ok NULL: none
struct DenseRows {
    const uint64_t *comp = nullptr;
    const uint32_t *pos = nullptr;
    const uint32_t *ok = nullptr;
};
// d_out -> int64 docIds (-1) and float distances (NaN) for empty or NaN entries; d_counts (nullable) [nq] real entries per query
cudaError_t launch_unpack_ragged(const RaggedBatch &b, const uint64_t *d_comp, uint32_t k, int64_t *d_labels, float *d_scores,
                                 uint32_t *d_counts, cudaStream_t s, LaunchCounters *ctr, const DenseRows &dense = DenseRows{});
// hybrid batches: bit `row` of d_bm[p] (words u32 per bitmap, zeroed) for every live entry of the list of query d_dense_q[p] whose
// docId maps to a row through d_table; one launch.  max_cap: the largest cap among those queries
cudaError_t launch_filter_bitmaps(const RaggedBatch &b, const uint32_t *d_dense_q, uint32_t n_dense, size_t max_cap, const uint32_t *d_table,
                                  uint32_t table_size, uint32_t *d_bm, uint32_t words, cudaStream_t s, LaunchCounters *ctr);
// hybrid batches: d_ok[q] = d_dense_ok[d_pos[q]] (0 for d_pos[q] == ~0: an ad-hoc query); d_live[q] = 0 for a proven query, else
// its live filter length; d_live_ptr[q] = d_live + q, the count table of the gather that answers the open queries
cudaError_t launch_hybrid_open(const RaggedBatch &b, const uint32_t *d_pos, const uint32_t *d_dense_ok, uint32_t *d_ok, uint32_t *d_live,
                               const uint32_t **d_live_ptr, cudaStream_t s, LaunchCounters *ctr);

// filter-set plumbing of the fused hybrid query: docId -> row id through a dense table; selected positions -> docIds
cudaError_t launch_map_labels(const uint32_t *d_labels, uint32_t n, const uint32_t *d_table, uint32_t table_size, uint32_t *d_ids,
                              cudaStream_t s, LaunchCounters *ctr);
cudaError_t launch_pick_labels(const uint64_t *d_comp, uint32_t k, const uint32_t *d_labels, uint32_t *d_out, cudaStream_t s,
                               LaunchCounters *ctr);

// ---- result unpacking / shard merge -------------------------------------------------------------
// composites [nq][k] + id->label table -> labels (int64, -1 for empty) and float scores.
cudaError_t launch_unpack_results(const uint64_t *d_comp, uint32_t nq, uint32_t k,
                                  const uint64_t *d_id_to_label, int64_t *d_labels, float *d_scores,
                                  cudaStream_t s, LaunchCounters *ctr);
// [G][nq][k] (score,label) -> [nq][k] by (score asc, label asc); label -1 = empty.
// score_stride / label_stride: elements between consecutive shards' arrays (0 = nq*k, i.e. dense [G][nq][k]).
cudaError_t launch_merge_shards(const float *d_scores, const int64_t *d_labels, uint32_t G, uint32_t nq,
                                uint32_t k, float *d_out_scores, int64_t *d_out_labels, cudaStream_t s,
                                LaunchCounters *ctr, size_t score_stride = 0, size_t label_stride = 0);
// G counted exchange blocks, block_bytes apart (layout: VecSimB200_ShardListBlockBytes) -> the merged [nq][w] rows and counts
// (DESIGN.md §6.1).  range: the cap rule of the range calls; by_id: runs ordered by label (range rows only).  One launch.
constexpr uint32_t kMaxListWidth = 4096;
cudaError_t launch_merge_lists(const void *d_blocks, size_t block_bytes, uint32_t G, uint32_t nq, uint32_t w, bool range, bool by_id,
                               int64_t *d_out_labels, float *d_out_scores, uint32_t *d_out_counts, cudaStream_t s, LaunchCounters *ctr);

} // namespace rsb200
