// Launchers of the posting-list kernels (ii_kernels.cu).  Plain CUDA runtime types only.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace rsb200 {

constexpr int kIIThreads = 256;
constexpr int kIIItems = 4;
constexpr int kIIChunk = kIIThreads * kIIItems; // entries of the driving list per CTA
constexpr int kIISmemElems = 8192;              // 32 KB window of the probed list staged per CTA
constexpr int kIIMaxLists = 32;        // children of one AND (kernel argument tables)
constexpr int kIIMaxUnionLists = 1024; // children of one OR: a prefix / fuzzy / wildcard expansion is a union of up to MAXEXPANSIONS
                                       // (default 200) terms; the union kernels take one list per launch and need no tables
constexpr int kIIUnionFlatMax = 20;    // above it the reference's union is UnionHeap (min_union_iter_heap, union_reducer.rs:106)

struct IntersectArgs {
    const uint32_t *ids[kIIMaxLists]; // [0] = the shortest list (drives), others ascending by length
    uint32_t len[kIIMaxLists];
    uint8_t mode[kIIMaxLists]; // per list (slot 0 = the driver, always required): 0 = required (AND), 1 = NOT (the docId must be
                               // absent: not.rs as a child of an intersection), 2 = OPTIONAL (never rejects: optional.rs)
    uint32_t n;
    uint32_t *tmp_idx;  // [nchunks*kIIChunk] survivors of chunk c at tmp_idx[c*kIIChunk + r] (index into list 0)
    uint32_t *tmp_pos;  // [n][stride]: position of entry idx of list 0 inside list j (valid for survivors)
    uint32_t *counts;   // [nchunks]
    size_t stride;      // nchunks*kIIChunk
};

struct GatherArgs {
    const uint32_t *ids0;
    const uint32_t *freqs[kIIMaxLists];
    uint8_t mode[kIIMaxLists]; // as IntersectArgs: NOT children yield freq 0, OPTIONAL children freq 0 where absent (virtual results)
    uint32_t n;
    const uint32_t *tmp_idx, *tmp_pos, *counts, *offsets;
    size_t stride;   // of tmp_pos
    uint32_t *out_doc;
    uint8_t row[kIIMaxLists]; // kernel slot j -> its row of out_freq / out_pos: the AGGREGATE child index
    uint32_t *out_freq; // [n][fstride]
    uint32_t *out_pos;  // nullable, [n][fstride]: position of the hit inside the child (phrase checks and GetSlop read the term
                        // positions there); 0xFFFFFFFF = a virtual result (NOT child / absent OPTIONAL child)
    size_t fstride;
};

// phrase constraints (slop / in-order): the term positions of every hit, children in aggregate order
constexpr int kPhraseMaxLists = 8;
struct PhraseArgs {
    const uint8_t *bytes[kPhraseMaxLists];    // gathered block bytes of list j (the offsets payloads live inside)
    const uint32_t *off_pos[kPhraseMaxLists]; // per posting: start of its offsets payload in bytes[j]
    const uint32_t *off_len[kPhraseMaxLists]; // per posting: length (0 / NULL array = the child carries no offsets)
    const uint32_t *pos;                      // [n][fstride] posting position of hit o inside child j (GatherArgs::out_pos)
    size_t fstride;
    uint32_t n;
    uint32_t max_slop; // 0xFFFFFFFF = no limit
    int in_order;
};
// survivors are compacted in order: docs, the n freq rows and (when d_out_pos is given) the n rows of a.pos
cudaError_t ii_launch_phrase_filter(const PhraseArgs &a, const uint32_t *d_len, uint32_t cap_len, uint32_t *d_flags, uint32_t *d_counts,
                                    uint32_t *d_offsets, uint32_t *d_total, const uint32_t *d_docs, const uint32_t *d_freqs, size_t fstride,
                                    uint32_t *d_out_docs, uint32_t *d_out_freqs, uint32_t *d_out_pos, size_t out_fstride, cudaStream_t s);

// GetSlop of the legacy scorers = IndexResult_MinOffsetDelta (src/index_result/index_result.c:51-108), one thread per hit.
// Rows of `pos` are in AGGREGATE child order: the posting position of the hit inside child j, 0xFFFFFFFF = the child is a
// virtual result here (NOT / absent OPTIONAL child of an intersection) or, for a union, is not part of the aggregate at all.
struct SlopArgs {
    const uint8_t *bytes[kIIMaxLists];
    const uint32_t *off_pos[kIIMaxLists];
    const uint32_t *off_len[kIIMaxLists]; // NULL: the child carries no offsets
    const uint32_t *pos;                  // [n][fstride]
    const struct UnionOrder *order;       // unions: the children in the reference's active-array order (NULL: index order)
    size_t fstride;
    uint32_t n;
    int is_union;
};
cudaError_t ii_launch_min_offset_delta(const SlopArgs &a, const uint32_t *d_docs, const uint32_t *d_len, uint32_t cap_len,
                                       uint32_t *d_slop, cudaStream_t s);

// ---- nested aggregates as children ------------------------------------------------------------------------------------
// freq of an aggregate result = the sum of its children's (RSAggregateResult push: result.freq += child.freq)
cudaError_t ii_launch_sum_freq_rows(const uint32_t *d_freqs, uint32_t n, size_t fstride, const uint32_t *d_len, uint32_t cap_len,
                                    uint32_t *d_out, cudaStream_t s);
// Term positions of an aggregate = the k-way merge of its children's offset iterators, duplicates kept
// (src/offset_vector.c:216-239 _aoi_Next, RS/index_result/src/core/proximity.rs:53-67 OffsetIter::Merge).  The merged stream of
// every hit is re-encoded as varint deltas so that the aggregate then looks like a term leaf to the phrase filter and to GetSlop:
// d_off_pos[o] / d_off_len[o] delimit it inside d_bytes.  Bit 31 of d_off_len[o] says the aggregate COUNTS as having offsets
// (by the kind mask of its children at this document, index_result.c:23-35 — even when the stream is empty).
constexpr uint32_t kIIOffLenHas = 0x80000000u;
struct MergeOffsetsArgs {
    const uint8_t *bytes[kIIMaxLists];
    const uint32_t *off_pos[kIIMaxLists];
    const uint32_t *off_len[kIIMaxLists]; // NULL: the child carries no offsets
    uint8_t tag[kIIMaxLists];             // RSResultData tag of the child's results: 1 union, 2 intersection, 4 term, 8 virtual, 16 numeric
    const uint32_t *pos;                  // [n][fstride], may be NULL (then presence comes from the freq rows)
    const uint32_t *freqs;                // [n][fstride]
    size_t fstride;
    uint32_t n;
    int is_union;
};
// pass 1: d_ub[o] = upper bound of the merged stream's bytes (the sum of the children's), per 256-hit chunk sums, their exclusive
// scan and the grand total (64-bit); pass 2 writes the streams (d_off_pos[o] = chunk offset + scan of d_ub inside the chunk)
cudaError_t ii_launch_merge_offsets_bounds(const MergeOffsetsArgs &a, const uint32_t *d_len, uint32_t cap_len, uint32_t *d_ub,
                                           uint32_t *d_chunk_sum, uint32_t *d_chunk_off, uint32_t *d_total32,
                                           unsigned long long *d_total64, cudaStream_t s);
cudaError_t ii_launch_merge_offsets_write(const MergeOffsetsArgs &a, const uint32_t *d_len, uint32_t cap_len, const uint32_t *d_ub,
                                          const uint32_t *d_chunk_off, uint8_t *d_bytes, uint32_t *d_off_pos, uint32_t *d_off_len,
                                          cudaStream_t s);

// UnionFlat keeps its children in an "active" array and swap-removes a child when it is exhausted (union_flat.rs:174-180,
// advance_and_find_min :218-258): the aggregate's child order for a document is the active array's order at that moment.
// For a union read front to back that order is a function of the docId alone: epoch e covers docIds in (bound[e-1], bound[e]].
struct UnionOrder {
    uint32_t n_epochs;
    uint32_t bound[kIIMaxLists + 1];
    uint8_t n_active[kIIMaxLists + 1];
    uint8_t perm[kIIMaxLists + 1][kIIMaxLists];
};

// ---- batches of ORs and numeric range filters (II_UnionBatchDevice, II_NumericFilterBatchDevice, II_UnionFilterBatchDevice) --
// Every list of every query of the batch in one ragged launch per step: each query owns a window of a shared bitmap that spans
// the docIds of its lists, a CTA of the mark / fill passes owns kUBChunk postings of one list (found by binary search over the
// lists' first chunks), and the scan runs one CTA per query.  Launches: 4 (docIds only) or 6 (per-child freq rows), whatever
// the batch size and the number of lists.  A set child's chunks are counted from its capacity; those past its count on the device
// return at once.
constexpr uint32_t kUBChunk = 1024;
struct UBList {
    const uint32_t *ids;
    const uint32_t *freqs; // full mode: the list's freqs (else NULL)
    const double *values;  // a numeric leaf: its record values, tested against the query's range (NULL: a posting list)
    const uint32_t *d_len; // a set: its count on the device, read as min(*d_len, len) (NULL: a list or a leaf, len is exact)
    uint32_t len;          // a list's or a leaf's length, a set's capacity
    uint32_t q;      // owning query (index into the UBQuery table)
    uint32_t row;    // the list's child index inside its query: its freq / position row
    uint32_t chunk0; // first kUBChunk chunk of the list in the batch
};
struct UBQuery {
    uint32_t *docs;  // the set's docIds [cap]
    uint32_t *freqs; // full mode: [n_rows][cap] (else NULL)
    uint32_t *pos;   // [n_rows][cap] posting position of the hit inside each child, ~0 = absent (NULL: not kept)
    uint32_t *len;   // [0] = the count; [1] = in-range records that are the first of their document in their leaf (numeric)
    UnionOrder *order;           // the set's epoch table (NULL: none) ...
    const UnionOrder *order_src; // ... copied from the uploaded batch table by the scan
    uint64_t blk0;     // first 32-word block of the query's window in the batch bitmap
    uint32_t nblk;     // blocks of the window
    uint32_t lo_word;  // the window covers docIds lo_word * 32 .. (lo_word + nwords) * 32 - 1
    uint32_t nwords;
    uint32_t n_rows;
    uint64_t cap;      // row stride of freqs / pos
    double mn, mx;     // numeric range (NumericFilter::value_in_range)
    int mni, mxi;
    // an OR over sets (sum_est = 1): len[1] = min(est_host + the sum of *est_dev[0 .. n_est_dev), 2^32 - 1), the children's
    // num_estimated with those still on the device read there; sum_est = 0: len[1] = the mark pass's count (numeric) or 0
    const uint32_t *const *est_dev;
    uint64_t est_host;
    uint32_t n_est_dev;
    uint32_t sum_est;
};
// d_est [nq] and d_bitmap [total_blocks * 32] are contiguous (one memset clears both); d_wordoff NULL = docIds only.
// clear_elems: the largest n_rows * cap of the batch (sizes the clear of the freq / position rows).  Returns the launches made.
cudaError_t ii_launch_union_batch(const UBList *d_lists, uint32_t nlists, uint32_t total_chunks, const UBQuery *d_q, uint32_t nq,
                                  uint64_t total_blocks, uint64_t clear_elems, uint32_t *d_est, uint32_t *d_bitmap, uint32_t *d_blocksum,
                                  uint32_t *d_blockoff, uint32_t *d_wordoff, uint32_t *launches, cudaStream_t s);

// ---- batches of filter-mode ANDs over lists and (pending) sets (II_IntersectFilterBatchDevice) ----------------------------
// A child is a posting list (exact length) or a set whose count is read on the device.  Each query's children sit in the child
// table in probe order: the driver first, then the others by ascending host bound.
struct IFBChild {
    const uint32_t *ids;
    const uint32_t *d_len; // a set: its count on the device, read as min(*d_len, len) (NULL: a list, len is exact)
    const uint32_t *d_est; // a set whose num_estimated is still on the device (NULL: `est` holds it)
    uint32_t len;          // a list: its length; a set: its capacity
    uint32_t est;          // num_estimated, saturated at 2^32 - 1
    uint32_t slot;         // the child's index in the order the caller gave (its estimate lands in len[2 + slot])
    uint32_t mode;         // 0 required, 1 NOT (an empty NOT child: len 0, ids NULL)
};
struct IFBQuery {
    uint32_t *docs;   // the set's docIds [cap]
    uint32_t *len;    // [0] the count, [1] num_estimated (the smallest required child's), [2 + i] child i's num_estimated
    uint32_t child0;  // first entry of the query in the child table: the driver
    uint32_t n;       // children
    uint32_t chunk0;  // first kIIChunk chunk of the driver in the batch
    uint32_t nchunks; // chunks of the driver (by its host bound)
};
// 3 launches whatever the batch: probe (one CTA per driver chunk, survivors compacted into d_surv[chunk * kIIChunk ...] and
// counted into d_counts), scan (one CTA per query: offsets, count, estimates), expand (one CTA per chunk: survivors to docs).
cudaError_t ii_launch_filter_and_batch(const IFBChild *d_children, const IFBQuery *d_q, uint32_t nq, uint32_t total_chunks,
                                       uint32_t *d_surv, uint32_t *d_counts, uint32_t *d_offsets, cudaStream_t s);

struct ScoreArgs {
    int scorer; // II_Scorer numbering
    int is_union;
    uint32_t n_children;
    double weight[kIIMaxLists], idf[kIIMaxLists], bm25_idf[kIIMaxLists]; // aggregate child order
    double agg_weight, avg_doc_len, min_score;
    uint64_t tanh_factor;
    const uint32_t *doc_len;   // by docId, may be NULL
    const float *doc_score;    // by docId, may be NULL
    const uint32_t *max_freq;  // by docId, may be NULL
    // GetSlop of the legacy scorers (BM25, TFIDF, TFIDF.DOCNORM divide by it): per hit when term positions are on the device,
    // else the value IndexResult_MinOffsetDelta returns without offsets: children - 1 (1 for a single child)
    const uint32_t *slop;      // per hit, may be NULL
    const UnionOrder *order;   // unions: child order per docId epoch (device memory), may be NULL
    const double *ext;         // more than kIIMaxLists children (unions): weight[n], idf[n], bm25_idf[n] in device memory instead of
                               // the inline tables above
    // NESTED aggregates (a child that is itself an evaluated AND / OR): sub[c] = the child's recursive score per hit OF THE
    // CHILD (what tfidfRecursive / bm25Recursive / bm25StdRecursive / dismaxRecursive return for it, its own weight applied:
    // src/ext/default.c:75-95,183-199,272-289,393-438), looked up through the hit's position inside the child
    const double *sub[kIIMaxLists]; // NULL: a leaf
    const uint32_t *pos;            // [n_children][pstride] position of the hit inside child c (0xFFFFFFFF: absent / virtual)
    size_t pstride;
    int sub_only;                   // 1: write the recursive value of THIS aggregate (no document-level factor): it is a nested child
};

// ---- fused batch search: AND + scorer + top-N of MANY queries in two launches --------------------------------------
constexpr int kFusedMaxLists = 8;   // more children: the per-query kernel chain
constexpr int kFusedMaxTopN = 128;
// One query of the batch.  Children are in the reference's aggregate order (ascending num_estimated, stable:
// RS/rqe_iterators/src/intersection.rs:110-145), and child 0 drives.  A field-mask-filtered child keeps its unfiltered
// estimate, so child 0 is not always the shortest list: the host sizes the batch from child 0 (fused_batch).
struct FusedQuery {
    const uint32_t *ids[kFusedMaxLists];
    const uint32_t *freqs[kFusedMaxLists];
    uint32_t len[kFusedMaxLists];
    double weight[kFusedMaxLists], idf[kFusedMaxLists], bm25_idf[kFusedMaxLists];
    uint32_t n;       // children (1..kFusedMaxLists)
    uint32_t item0;   // first work item (1024-entry chunk of child 0) of this query in the batch
    uint32_t nchunks; // work items of this query
    uint32_t _pad;
};
struct FusedCommon {
    int scorer;
    double agg_weight, avg_doc_len;
    uint64_t tanh_factor;
    const uint32_t *doc_len;
    const float *doc_score;
    const uint32_t *max_freq;
};
// Launches: (1) item -> query table; (2) one thread per (work item, other child): the window of the child that can hold the
// item's docIds; (3) one CTA per work item — every window staged in shared memory at once (list by list when they do not fit),
// membership, freqs of the matches, the scorer, and the CTA's best `top_n` hits into cand_keys / cand_ids [item][top_n] (padded
// with ~0); hits[q] += survivors; (4) one CTA per query selects the best top_n by (score desc, docId asc) over its items'
// candidates into out_keys / out_ids [nq][top_n].  d_item_q: [total_items]; d_win: [total_items][kFusedMaxLists - 1];
// d_hits: [2 * nq] (survivors per query, then the fill level of each query's compact candidate list).
cudaError_t ii_launch_fused_search(const FusedQuery *d_queries, uint32_t nq, uint32_t total_items, uint32_t max_children, const FusedCommon &fc,
                                   uint32_t top_n, uint32_t *d_item_q, uint2 *d_win, uint64_t *d_cand_keys, uint32_t *d_cand_ids,
                                   uint32_t *d_hits, uint64_t *d_out_keys, uint32_t *d_out_ids, cudaStream_t s);

cudaError_t ii_launch_decode(const uint8_t *d_bytes, const uint64_t *d_byte_off, const uint64_t *d_first_id,
                             const uint32_t *d_entry_off, uint32_t nblocks, int codec, uint64_t wide_filter_lo, uint64_t wide_filter_hi,
                             uint32_t *d_ids, uint32_t *d_freqs, uint32_t *d_masks, cudaStream_t s);
// batch decode: 32-bit tables (byte_off[nblocks+1] into the 16-byte-aligned, 16-byte-padded gathered stream, first_id[nblocks],
// entry_off[nblocks+1] into the output arrays), blocks of MANY lists back to back
cudaError_t ii_launch_decode_staged(const uint8_t *d_bytes, const uint32_t *d_byte_off, const uint32_t *d_first_id,
                                    const uint32_t *d_entry_off, uint32_t nblocks, int codec, uint32_t *d_ids, uint32_t *d_freqs,
                                    uint32_t *d_masks, uint32_t *d_off_pos, uint32_t *d_off_len, cudaStream_t s);
// numeric index (RS/inverted_index/src/codec/numeric.rs): blocks -> (docId u32, value f64); range filter -> ordered docIds, one per
// document (freq 1)
cudaError_t ii_launch_decode_numeric(const uint8_t *d_bytes, const uint64_t *d_byte_off, const uint64_t *d_first_id, const uint32_t *d_entry_off,
                                     uint32_t nblocks, uint32_t *d_ids, double *d_values, cudaStream_t s);
cudaError_t ii_launch_numeric_filter(const uint32_t *d_ids, const double *d_values, uint32_t n, double mn, double mx, bool min_inclusive,
                                     bool max_inclusive, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_total, uint32_t *d_out_ids,
                                     uint32_t *d_out_freqs, cudaStream_t s);
cudaError_t ii_launch_mask_filter(const uint32_t *d_ids, const uint32_t *d_freqs, const uint32_t *d_masks, uint32_t n,
                                  uint32_t filter, uint32_t *d_counts, uint32_t *d_offsets, uint32_t *d_total,
                                  uint32_t *d_out_ids, uint32_t *d_out_freqs, cudaStream_t s);
cudaError_t ii_launch_intersect(const IntersectArgs &a, uint32_t nchunks, uint32_t *d_offsets, uint32_t *d_total,
                                cudaStream_t s);
cudaError_t ii_launch_gather(const GatherArgs &g, uint32_t nchunks, cudaStream_t s);
cudaError_t ii_launch_score(const ScoreArgs &sa, const uint32_t *d_docs, const uint32_t *d_freqs, size_t fstride,
                            const uint32_t *d_len, uint32_t cap_len, double *d_scores, cudaStream_t s);
cudaError_t ii_launch_union(const uint32_t *const *d_ids, const uint32_t *const *d_freqs, const uint32_t *lens, uint32_t n,
                            uint32_t nwords, uint32_t *d_bitmap, uint32_t *d_blocksum, uint32_t *d_blockoff,
                            uint32_t *d_wordoff, uint32_t *d_total, uint32_t *d_out_doc, uint32_t *d_out_freq,
                            size_t fstride, bool want_freqs, uint32_t *d_out_pos, cudaStream_t s);
// HAMMING scorer (src/ext/default.c:475-497): 1 / (popcount(query payload XOR document payload) + 1); 0 when the document has no
// payload or the lengths differ.  payload_off[d] .. payload_off[d+1] delimit the payload of docId d inside `payloads`.
cudaError_t ii_launch_hamming(const uint32_t *d_docs, const uint32_t *d_len, uint32_t cap_len, const uint8_t *d_payloads,
                              const uint64_t *d_payload_off, const uint8_t *d_qdata, uint32_t qlen, double *d_scores, cudaStream_t s);
cudaError_t ii_launch_iota(uint32_t *d_ids, uint32_t *d_freqs, uint32_t n, cudaStream_t s);
uint32_t ii_topn_lists(uint32_t m);
cudaError_t ii_launch_topn(const uint32_t *d_docs, const double *d_scores, const uint32_t *d_len, uint32_t cap_len, uint32_t k,
                           uint64_t *d_keys, uint32_t *d_ids, cudaStream_t s);

} // namespace rsb200
