// Launchers of the tensor-core coarse pass (coarse_tc.cu): wgmma GEMM (fp16 shadow rows or TF32 on the
// fp32 rows) with fused candidate selection, exact rescoring, and the completeness proof.  See the header
// comment of coarse_tc.cu.
#pragma once
#include "vecsim_kernels.h"

namespace rsb200 {

constexpr uint32_t kCoarseKeep = 24;       // candidates kept per (CTA row range, query), first tier
constexpr uint32_t kCoarseKeepWide = 128;  // second tier (queries the first proof left open) and first tier of k > 16
constexpr uint32_t kCoarseTier1MaxK = 16;  // largest k the 24-entry lists serve
constexpr uint32_t kCoarseMaxK = 128;      // largest k served by the coarse path (TF32, direct 16/8-bit routes, tier 1 at small k)
constexpr uint32_t kCoarseMaxKWide = 1024; // largest k of the fp32 route's two-pass first tier (DESIGN.md §4.5)
constexpr uint32_t kCoarseFixedCapWide = 256; // list capacity of the fp32 main pass for k > kCoarseMaxK
constexpr uint32_t kCoarseSampleSlices = 32; // minima the sample pass publishes per (query, row range)
constexpr uint32_t kCoarseFixedCapDirect = 256; // list capacity of the fixed-bound pass on 16-bit corpora (k up to 128)
constexpr uint32_t kCoarseFixedCapQ8 = 256;   // list capacity of the main pass over the int8 shadow (its bound admits more rows)
constexpr uint32_t kCoarseFixedCap = 96;   // list capacity of the fixed-bound main pass (rows below the bound per row range)
constexpr uint32_t kRangeFoldMaxHits = 4096; // most hit rows range_label_fold_kernel sorts per query (48 KB of shared memory)
// |approx - exact| bounds for unit vectors (Cauchy-Schwarz over the dot product: sum |a_i b_i| <= 1):
//  TF32: each operand truncated to 11 significant bits -> 2 * 2^-10 relative per product, + accumulation slack;
//  F16 : each operand rounded to nearest, 11 significant bits -> 2 * 2^-11 = 9.8e-4 per product; elements below
//        the fp16 normal range (6.1e-5) add at most 2^-25 * sum|b_i| <= 2^-25 * sqrt(dim) <= 1e-6; fp32
//        accumulation of <= 1024 terms adds < 1.3e-4.
constexpr float kCoarseEpsTF32 = 2.5e-3f;
constexpr float kCoarseEpsF16 = 1.2e-3f;

// CoarseQ8: the int8 shadow of fp32 unit rows (cosine, k <= kCoarseMaxK), one scale per 128-row tile, error bound per query
enum CoarseKind : int { CoarseTF32 = 0, CoarseF16 = 1, CoarseDirect16 = 2, CoarseDirect8 = 3, CoarseQ8 = 4 };
inline float coarse_eps(CoarseKind k) { return k == CoarseF16 ? kCoarseEpsF16 : kCoarseEpsTF32; }

struct CoarsePlan {
    CoarseKind kind;
    uint32_t grid_x, grid_y, num_kb, tiles, keep;
    uint32_t stages; // depth of the row-tile ring in shared memory
    uint32_t threads; // block size of the kernel the plan launches
    uint32_t epl;    // candidate-list entries per lane of the compacting warp (3 or 8)
    uint32_t tile_stride; // 1 = every row tile; n = every n-th (the sample pass)
    int mode;        // CoarseF16: 0 adaptive top-`keep` lists, 1 fixed admission bound per query (main pass), 2 sample pass (slice minima)
    uint32_t csize;  // thread-block cluster size along y (query groups sharing multicast row tiles); 1 = none
    uint32_t reg_kb; // CoarseF16 mode 1: leading K blocks of the resident queries held in registers (0 = all in shared memory)
    size_t cand_elems; // uint64 per (query, list, keep)
    size_t scratch_elems; // uint64 of per-CTA candidate-list scratch (CoarseF16), 0 otherwise
    size_t smem_bytes;
};

// operands of the coarse GEMM in the element type of `kind`: corpus rows and the query batch
struct CoarseOperands {
    const void *rows;
    size_t pitch;
    const void *queries;
    size_t qpitch;
    int elem_variant; // CoarseDirect16: 1 = bfloat16 (else IEEE half); CoarseDirect8: 1 = int8 (else uint8)
    int epilogue;     // CoarseDirect8: 0 inner product, 1 cosine (rows carry their fp32 norm after the payload), 2 squared L2
                      // (needs the two arrays below, as int32); CoarseF16: 1 = squared-L2 epilogue (needs the two arrays below)
    const float *row_norm2; // CoarseF16 / L2: |row|^2 per row (fp32 rows); CoarseDirect8 / L2: exact int32 |row|^2 per row
    const float *q_norm2;   //                 |q|^2 per query;                CoarseDirect8 / L2: exact int32 |q|^2 per query
};
bool coarse_supported(const CorpusView &c, uint32_t nq, uint32_t k, CoarseKind kind);
// keep_override != 0 (CoarseF16 only): candidates per list instead of the default for k.  filt: the pass is launched with row
// filters (launch_coarse's d_filt)
CoarsePlan plan_coarse(const CorpusView &c, uint32_t nq, CoarseKind kind, uint32_t k, uint32_t keep_override = 0, uint32_t tile_stride = 1,
                       int mode = 0, bool filt = false);
// d_nq_dev (nullable): the number of live queries is read from device memory (min with nq); 0 = the kernel exits at once.
// d_filt (nullable; CoarseF16, and CoarseDirect8 of mode 1): row filters of a hybrid batch, one bitmap of filt_words u32 per query
// (bit r = row r); query i of the pass uses bitmap d_filt_q[i] (d_filt_q NULL: bitmap i).  Only filtered rows enter the lists and
// the sample minima.  d_list_count (nullable; mode 1): [nq][grid_x], the entries of each published list.  Required by the fixed
// pass over the int8 shadow (CoarseQ8, mode 1), whose lists carry those entries only, with no kEmptySlot padding
cudaError_t launch_coarse(const CoarseOperands &o, uint32_t n_rows, uint32_t dim, uint32_t nq, const CoarsePlan &p, uint64_t *d_cand,
                          uint64_t *d_scratch, cudaStream_t s, const uint32_t *d_nq_dev = nullptr, const float *d_thr_fixed = nullptr,
                          uint32_t *d_overflow = nullptr, const uint32_t *d_filt = nullptr, uint32_t filt_words = 0,
                          const uint32_t *d_filt_q = nullptr, uint32_t *d_list_count = nullptr);
// bound of the fixed pass from the sample pass's candidate lists: d_thr[q] = k-th smallest approximate distance + 2 eps;
// clears d_overflow[q].  d_q_eps (nullable; the int8 shadow): eps of each query, in place of eps / d_q_norm2
cudaError_t launch_threshold(const uint64_t *d_cand, uint32_t nq, uint32_t lists_per_query, uint32_t keep, uint32_t k, float eps,
                             const float *d_q_norm2, float max_norm, uint32_t dim, int l2, float *d_thr, uint32_t *d_overflow, cudaStream_t s,
                             const float *d_q_eps = nullptr);
// fp32 rows [first, first+n) -> the tiled fp16 shadow copy read by the CoarseF16 kernel (layout in coarse_tc.cu);
// the buffer holds coarse_shadow_bytes(capacity_rows, dim) bytes
size_t coarse_shadow_bytes(uint32_t rows, uint32_t dim);
cudaError_t launch_to_f16_tiled(const void *src, size_t spitch, uint32_t dim, uint32_t first, uint32_t n, void *dst, cudaStream_t s);
// fp32 unit rows -> the tiled int8 shadow read by the CoarseQ8 kernel: every 128-row tile that holds a row of [first, first+n) is
// quantized whole (rows past n_rows are zero) with its scale s_t = max |x| / 127 into d_tscale[tile], round to nearest.  d_stats
// keeps running maxima, as float bits rounded up, of the residual norm |x - s_t x~| and of |x| over the rows quantized; the buffer
// holds coarse_shadow8_bytes(capacity_rows, dim) bytes
size_t coarse_shadow8_bytes(uint32_t rows, uint32_t dim);
cudaError_t launch_to_i8_tiled(const void *src, size_t spitch, uint32_t dim, uint32_t n_rows, uint32_t first, uint32_t n, void *dst,
                               float *d_tscale, uint32_t *d_stats, cudaStream_t s);
// bytes of one int8 query row of the CoarseQ8 kernel: the payload padded to 16, its scale s_q (float), padding
inline size_t coarse_q8_payload(uint32_t dim) { return (dim + 15) & ~(size_t)15; }
inline size_t coarse_q8_pitch(uint32_t dim) { return coarse_q8_payload(dim) + 16; }
// nq fp32 unit queries -> int8 rows (coarse_q8_pitch) with their scale, and d_eps[q], a rigorous bound of |approx - exact| for
// every stored row, from the row bounds delta_max (residual norm) and x_max (row norm) of the shadow; NaN when not finite
cudaError_t launch_quantize_queries(const void *d_q, size_t qpitch, uint32_t dim, uint32_t nq, void *d_q8, float *d_eps, float delta_max,
                                    float x_max, cudaStream_t s);
// fp32 rows [first, first+n) -> row-major fp16 rows (the query batch; dim % 8 == 0)
cudaError_t launch_to_f16(const void *src, size_t spitch, uint32_t dim, uint32_t first, uint32_t n, void *dst, size_t dpitch,
                          cudaStream_t s);
// One CTA per query: exact rescoring of the candidates within 2 eps of the k-th best approximate distance, exact top-k
// (d_out[q][k], ascending, kEmptySlot padded) and the completeness proof (d_ok[q]).  d_q_norm2 == NULL: unit vectors,
// |approx - exact| <= eps; otherwise the bound scales with max_norm (over all rows) and |q| (refine_kernel).  Second tier:
// d_q_index[i] = query of the original batch whose lists sit at position i (d_q_norm2 is indexed by position), *d_nq_dev
// live positions.  d_row_label (nullable): the answer's composites carry row_label[row] (a docId) in place of the row, and ties
// resolve by it.  d_q_eps (nullable; the int8 shadow): the bound of each query by position, in place of eps / d_q_norm2.
// d_list_count (nullable; with d_thr_T): [nq][lists_per_query] entries of each list (launch_coarse's d_list_count), which
// are read instead of the kEmptySlot padding.
cudaError_t launch_refine(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t lists_per_query, uint32_t keep,
                          uint32_t k, const uint64_t *d_cand, float eps, const float *d_q_norm2, float max_norm, uint32_t *d_ok,
                          uint64_t *d_out, const uint32_t *d_q_index, const uint32_t *d_nq_dev, cudaStream_t s,
                          const float *d_thr_T = nullptr, const uint32_t *d_overflow = nullptr, const uint64_t *d_row_label = nullptr,
                          const float *d_q_eps = nullptr, const uint32_t *d_list_count = nullptr);
// direct 16-bit route: d_ok[q] = d_overflow[q] ? 0 : 1
cudaError_t launch_flags_from_overflow(const uint32_t *d_overflow, uint32_t nq, uint32_t *d_ok, cudaStream_t s);
// second tier of the direct route: row i of src ([.][k] composites) -> row d_idx[i] of dst, d_ok[d_idx[i]] = 2, for i < *d_count
cudaError_t launch_scatter_rows(const uint64_t *d_src, const uint32_t *d_idx, const uint32_t *d_count, uint32_t max_n, uint32_t k,
                                uint64_t *d_dst, uint32_t *d_ok, cudaStream_t s);
// d_idx[0, *d_count) = the queries with d_ok == 0, ascending
cudaError_t launch_compact_unproven(const uint32_t *d_ok, uint32_t nq, uint32_t *d_idx, uint32_t *d_count, cudaStream_t s);
// row i of dst = row d_idx[i] of src (pitch % 16 == 0), squared norms likewise (nullable), for i < *d_count
cudaError_t launch_gather_queries(const void *d_src, size_t pitch, const float *d_src_n2, const uint32_t *d_idx, const uint32_t *d_count,
                                  uint32_t max_n, void *d_dst, float *d_dst_n2, cudaStream_t s);
// range batches: bound of the fixed-bound main pass, d_thr[q] = d_radius[q] + eps_q (rounded up); clears d_overflow[q] and
// *d_total
cudaError_t launch_range_bound(const float *d_radius, uint32_t nq, float eps, const float *d_q_norm2, float max_norm, uint32_t dim, int l2,
                               float *d_thr, uint32_t *d_overflow, uint32_t *d_total, cudaStream_t s);
// device range batches on fp16 / bf16 (dtype) inner product or cosine (the direct route, DESIGN.md §4.11): d_thr[q] = d_radius[q] +
// eps16_q rounded up, eps16_q from |q| of the stored query and max_norm = X, the running maximum row norm; -inf where |q|, X or the
// bound is not finite (the query is then never proven).  Clears d_overflow[q]
cudaError_t launch_range_bound16(const void *d_queries, size_t qpitch, uint32_t nq, uint32_t dim, int dtype, const float *d_radius,
                                 float max_norm, float *d_thr, uint32_t *d_overflow, cudaStream_t s);
// range batches, one CTA per query over its `slots` list entries of the main pass (d_cand, overwritten): exact rescoring and
// the inclusive test d <= d_radius[q].  Query q's hits go to d_out[d_off[q], d_off[q] + d_cnt[q]) (composites, unordered;
// d_out holds nq * slots); d_ok[q] = 1 if the answer is proven complete, else 0 with d_cnt[q] = 0.  d_q_norm2 == NULL: unit
// rows.  fp32 rows (L2 / inner product), or fp16 / bf16 rows (inner product) rescored with DistTile16.  cap != 0 (device range batches): query q's hits go to d_out[q * cap, q * cap + min(d_cnt[q], cap)) instead, d_cnt[q] the
// true count; d_total and d_off are not used.
cudaError_t launch_range_refine(const CorpusView &c, const void *d_queries, size_t qpitch, uint32_t nq, uint32_t slots, uint64_t *d_cand,
                                const float *d_radius, const float *d_q_norm2, const float *d_thr, const uint32_t *d_overflow, uint64_t *d_out,
                                uint32_t *d_total, uint32_t *d_ok, uint32_t *d_cnt, uint32_t *d_off, cudaStream_t s, uint32_t cap = 0);
// fixed-radius pass over 8-bit corpora (launch_coarse on a CoarseDirect8 plan of mode 1, d_thr_fixed = the radii): the real
// entries of query q's `slots` list entries -> d_out[q * cap, ...) unordered, d_cnt[q] = their number (past cap too), d_ok[q] = 1;
// a query whose lists overflowed: d_ok[q] = 0, d_cnt[q] = 0
cudaError_t launch_range_pack(const uint64_t *d_cand, uint32_t nq, uint32_t slots, const uint32_t *d_overflow, uint32_t cap, uint64_t *d_out,
                              uint32_t *d_cnt, uint32_t *d_ok, cudaStream_t s);
// device range batches on multi-value indexes (DESIGN.md §4.12): the label fold of the queries a route proved.  d_front != NULL (fp32
// route, after launch_range_refine with d_out = d_cand and cap = slots): query q's hit rows are d_cand[q * slots, + d_front[q]), proven
// iff d_ok[q] != 0; d_front == NULL (8-bit route, in place of launch_range_pack): its hits are the real entries of its `slots` list
// entries, proven iff d_overflow[q] == 0.  A proven query with at most kRangeFoldMaxHits hits gets one composite (score key, row)
// per label, the label's smallest (score, row), in d_out[q * cap, ...) unordered, d_cnt[q] = the number of labels (past cap too),
// d_ok[q] = d_flags[q] = 1.  With more hits: d_ok[q] = 0, d_flags[q] = 3; an unproven query: d_ok[q] = d_flags[q] = 0.  d_cnt[q]
// is left as it was (zero) for both.
cudaError_t launch_range_label_fold(const uint64_t *d_cand, uint32_t nq, uint32_t slots, const uint32_t *d_front, const uint32_t *d_overflow,
                                    const uint64_t *d_id_to_label, uint32_t cap, uint64_t *d_out, uint32_t *d_cnt, uint32_t *d_ok,
                                    uint32_t *d_flags, cudaStream_t s);
// |row|^2 of fp32 rows [first, first+n) into d_norm2[first..], NaN for a row whose fp16 form is not finite (a component
// with |x| >= 65520, or NaN: refine_kernel never proves such a query); d_stats (nullable) = {max |row|^2, max |x|} as float bits.
// dtype DT_F16 / DT_BF16: the same over stored 16-bit rows
cudaError_t launch_row_stats(const void *rows, size_t pitch, uint32_t dim, uint32_t first, uint32_t n, float *d_norm2, uint32_t *d_stats,
                             cudaStream_t s, int dtype = DT_F32);
// exact int32 |x|^2 of int8 (is_signed) / uint8 rows [first, first+n) into d_norm2[first..] (dim <= 2048: no overflow); serves
// the corpus rows and the query batch of the 8-bit L2 route
cudaError_t launch_int_norm2(const void *rows, size_t pitch, uint32_t dim, uint32_t first, uint32_t n, bool is_signed, int32_t *d_norm2,
                             cudaStream_t s);

} // namespace rsb200
