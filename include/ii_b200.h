/* ii_b200.h — C-ABI of libii_b200.so: posting-list intersection / union and BM25 / TF-IDF scoring on
 * B200, behind the reference's QueryIterator and scorer surfaces.
 *
 * How it slots under FT.SEARCH (details and the exact call sites in INTEGRATION.md):
 *   - term readers are opened by RediSearch as today; their IndexBlocks
 *     (RS/headers/inverted_index_ffi.h:102-132 IndexBlock_{Data,FirstId,LastId,NumEntries},
 *     :286 InvertedIndex_BlockRef) are handed to II_PostingList_FromBlocks, which decodes them on the
 *     host (all cores) or on the device and keeps (docId, freq) arrays resident in HBM;
 *   - where query evaluation would call NewIntersectionIterator / NewUnionIterator
 *     (RS/headers/iterators_ffi.h:309,594) over term leaves, it calls II_Intersect / II_Union; the whole
 *     iterator tree runs as a few kernels and yields an II_ResultSet of ascending docIds;
 *   - II_Score applies one of the reference's default scorers (src/ext/default.c) to every hit on
 *     device with the reference's exact expression trees;
 *   - II_NewResultIterator wraps the result set in an object whose first member is layout-identical
 *     to the reference's `QueryIterator` (src/iterators/iterator_api.h:46-151): Read / SkipTo / Rewind /
 *     NumEstimated / Revalidate / Free honour the contract at :88-117, and `current` points at a
 *     struct layout-identical to `RSIndexResult` (RS/headers/index_result_rs.h:584-621) carrying the
 *     docId and the pre-computed score as a Metric value, so RPScorer can return it unchanged
 *     (the "pre-score inside a custom iterator" route of SURVEY.md §8b).
 * Layouts are checked against tests/golden/ii_abi_layout.txt (generated from the reference headers).
 *
 * No CPU fallback: constructors return NULL when no CUDA device is usable.  docIds above 2^32-2 are
 * not representable on the device (t_docId is 64-bit in the reference; the BASELINE corpora are <= 50M).
 */
#ifndef II_B200_H
#define II_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint64_t t_docId;

/* ---- reference-compatible iterator surface (src/iterators/iterator_api.h) ------------------- */
typedef enum { ITERATOR_OK = 0, ITERATOR_NOTFOUND = 1, ITERATOR_EOF = 2, ITERATOR_TIMEOUT = 3 } IteratorStatus;
typedef enum { VALIDATE_OK = 0, VALIDATE_MOVED = 1, VALIDATE_ABORTED = 2, VALIDATE_TIMEOUT = 3 } ValidateStatus;
/* RS/headers/rqe_iterator_type.h */
enum { II_IteratorType_InvIdxWildcard = 2, II_IteratorType_Union = 6, II_IteratorType_Intersect = 7, II_IteratorType_Wildcard = 12,
       II_IteratorType_Empty = 13,
       II_IteratorType_MetricSortedById = 16 };
/* RS/headers/index_result_rs.h RawResultData_Active_Tag */
enum { II_ResultData_Union = 1, II_ResultData_Intersection = 2, II_ResultData_Term = 4, II_ResultData_Virtual = 8,
       II_ResultData_Numeric = 16, II_ResultData_Metric = 32 };

/* Layout-identical to RSIndexResult (112 bytes): docId@0 dmd@8 fieldMask@16 freq@32 data@40
 * metrics@80 weight@88 hasFieldExpiration@96. */
typedef struct II_IndexResult {
    t_docId docId;
    const void *dmd;            /* RSDocumentMetadata*, filled by RPQueryIterator's DocTable_Borrow */
    unsigned __int128 fieldMask; /* t_fieldMask */
    uint32_t freq;              /* aggregate freq = sum over matched children */
    struct {
        uint8_t tag;            /* II_ResultData_Metric */
        uint8_t _pad[7];
        double metric;          /* the pre-computed score (or 0 when unscored) */
        uint8_t _rest[24];
    } data;
    void *metrics;              /* MetricsVec: empty */
    double weight;
    bool hasFieldExpiration;
} II_IndexResult;

struct IndexSpec;
/* Layout-identical to QueryIterator (88 bytes). */
typedef struct II_QueryIterator {
    uint32_t type; /* enum IteratorType */
    bool atEOF;
    t_docId lastDocId;
    II_IndexResult *current;
    size_t (*NumEstimated)(const struct II_QueryIterator *self);
    IteratorStatus (*Read)(struct II_QueryIterator *self);
    IteratorStatus (*SkipTo)(struct II_QueryIterator *self, t_docId docId);
    ValidateStatus (*Revalidate)(struct II_QueryIterator *self, struct IndexSpec *spec);
    void (*Free)(struct II_QueryIterator *self);
    void (*Rewind)(struct II_QueryIterator *self);
    struct II_QueryIterator *(*ProfileChildren)(struct II_QueryIterator *self);
    void (*PrintProfile)(const struct II_QueryIterator *self, void *map, void *ctx);
} II_QueryIterator;

/* RSIndexStats (src/redisearch.h:245-249) */
typedef struct {
    size_t numDocs;
    size_t numTerms;
    double avgDocLen;
} II_IndexStats;

/* ---- posting lists ---------------------------------------------------------------------------- */
typedef enum {
    II_CODEC_FULL = 0,        /* qint4[delta,freq,fieldMask,offsetsLen]+offsets  RS/inverted_index/src/codec/full.rs:66-69 */
    II_CODEC_FREQS_ONLY = 1,  /* qint2[delta,freq]                               codec/freqs_only.rs:33 */
    II_CODEC_FREQS_FIELDS = 2,/* qint3[delta,freq,fieldMask]                     codec/freqs_fields.rs:43 */
    II_CODEC_FIELDS_ONLY = 3, /* qint2[delta,fieldMask]                          codec/fields_only.rs:43 */
    II_CODEC_DOCIDS_ONLY = 4, /* varint(delta)                                   codec/doc_ids_only.rs:33 */
    II_CODEC_RAW_DOCIDS_ONLY = 5, /* u32 (docId - block.first_doc_id)            codec/raw_doc_ids_only.rs:31-37 */
    II_CODEC_FREQS_OFFSETS = 6,   /* qint3[delta,freq,offsetsLen]+offsets            codec/freqs_offsets.rs:32-64 */
    II_CODEC_OFFSETS_ONLY = 7,    /* qint2[delta,offsetsLen]+offsets (freq 1)        codec/offsets_only.rs:31-62 */
    II_CODEC_FIELDS_OFFSETS = 8,  /* qint3[delta,fieldMask,offsetsLen]+offsets       codec/fields_offsets.rs:36-84 */
    /* u128 field masks (more than 32 fields), the mask as a varint after the qint group: */
    II_CODEC_FULL_WIDE = 9,           /* qint3[delta,freq,offsetsLen]+varint(mask)+offsets   codec/full.rs:197-232 */
    II_CODEC_FREQS_FIELDS_WIDE = 10,  /* qint2[delta,freq]+varint(mask)                      codec/freqs_fields.rs:114-145 */
    II_CODEC_FIELDS_ONLY_WIDE = 11,   /* varint(delta)+varint(mask)                          codec/fields_only.rs:109-137 */
    II_CODEC_FIELDS_OFFSETS_WIDE = 12 /* qint2[delta,offsetsLen]+varint(mask)+offsets        codec/fields_offsets.rs:138-185 */
} II_Codec;

/* One IndexBlock as the reference exposes it (RS/inverted_index/src/index/core.rs:76-94). */
typedef struct {
    uint64_t first_doc_id;
    uint64_t last_doc_id;
    uint16_t num_entries;
    const uint8_t *data;
    size_t len;
} II_BlockView;

typedef struct II_PostingList II_PostingList; /* (docId u32, freq u32) arrays resident in HBM */

/* Decode `nblocks` IndexBlocks into a device-resident posting list.  field_mask_filter != 0 keeps only
 * records with (fieldMask & filter) != 0, like FilterMaskReader (RS/inverted_index/src/reader/field_mask.rs);
 * the estimate reported to the intersection sort stays the unfiltered entry count.
 * decode_on_device: 0 = host decode on all cores then one H2D copy; 1 = ship the raw block bytes and
 * decode in a kernel (one thread per block). */
II_PostingList *II_PostingList_FromBlocks(const II_BlockView *blocks, size_t nblocks, II_Codec codec,
                                          uint32_t field_mask_filter, int decode_on_device);
/* The same with a 128-bit field-mask filter {low 64 bits, high 64 bits} for the *Wide codecs (t_fieldMask is u128 on 64-bit
 * builds of the reference); NULL or all zero = no filter.  A filter with bits above 31 on a 32-bit-mask codec is refused. */
II_PostingList *II_PostingList_FromBlocksWideMask(const II_BlockView *blocks, size_t nblocks, II_Codec codec, const uint64_t filter128[2],
                                                  int decode_on_device);
/* The same for MANY lists in one call (the terms of a batch of queries): one gather of all block bytes and block tables
 * into pinned staging, one H2D copy, one decode launch, one synchronisation; the lists share their device arrays.
 * blocks[i] / nblocks[i] describe list i, out[i] receives its handle (NULL if it could not be built).  Returns the number
 * of lists built. */
size_t II_PostingList_FromBlocksBatch(size_t n_lists, const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec,
                                      II_PostingList **out);
/* Same, and the TERM POSITIONS stay on the device (the codecs that store them: FULL, FREQS_OFFSETS, OFFSETS_ONLY, FIELDS_OFFSETS and
 * the wide variants; other codecs behave like the call above): the encoded
 * block bytes are kept resident and every posting records where its offsets payload (varint position deltas,
 * RS/index_result/src/core/proximity.rs:45-52) sits inside them.  Needed by slop / in-order intersections. */
size_t II_PostingList_FromBlocksBatchOffsets(size_t n_lists, const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec,
                                             II_PostingList **out);
int II_PostingList_HasOffsets(const II_PostingList *pl);
/* The index WRITER — InvertedIndex::add_record (RS/inverted_index/src/index/core.rs:235-358): 100 entries per block (1000 for the
 * docId-only codecs), delta from the previous docId (from the block's first docId for RawDocIdsOnly), a fresh block when the delta
 * does not fit the encoder, a repeated docId dropped (term codecs) or kept in the same block (numeric: multi-value documents).
 * The blocks are byte-identical to the reference's for the same records.  Host code; no device involved. */
typedef struct II_IndexWriter II_IndexWriter;
II_IndexWriter *II_IndexWriter_New(II_Codec codec);
II_IndexWriter *II_IndexWriter_NewNumeric(int compress_floats); /* Numeric / NumericFloatCompression */
/* bytes appended (0: the record was dropped).  mask = {lo, hi} halves of the u128 field mask; offsets = varint position deltas */
size_t II_IndexWriter_Add(II_IndexWriter *w, uint64_t doc_id, uint32_t freq, uint64_t mask_lo, uint64_t mask_hi, const uint8_t *offsets,
                          uint32_t offsets_len);
size_t II_IndexWriter_AddNumeric(II_IndexWriter *w, uint64_t doc_id, double value);
size_t II_IndexWriter_NumBlocks(const II_IndexWriter *w);
size_t II_IndexWriter_NumDocs(const II_IndexWriter *w); /* unique documents */
int II_IndexWriter_Block(const II_IndexWriter *w, size_t i, II_BlockView *out); /* valid until the next Add / Free */
void II_IndexWriter_Free(II_IndexWriter *w);

/* NUMERIC index blocks (the leaves of the reference's numeric range tree; RS/inverted_index/src/codec/numeric.rs: header byte,
 * 0-7 delta bytes, tiny / integer / f32 / f64 / infinite value; duplicates of a docId allowed = multi-value documents) decoded on
 * the device into (docId, value) arrays, and range filters over them (NumericFilter::value_in_range, reader/numeric.rs:80-85):
 * II_NumericList_Filter yields the matching docIds ascending, one per document, as a posting list (freq 1) that takes part in
 * AND / OR / hybrid pre-filters like a term leaf. */
typedef struct II_NumericList II_NumericList;
II_NumericList *II_NumericList_FromBlocks(const II_BlockView *blocks, size_t nblocks);
size_t II_NumericList_Len(const II_NumericList *nl);
int II_NumericList_Fetch(const II_NumericList *nl, uint64_t *doc_ids, double *values); /* either may be NULL */
II_PostingList *II_NumericList_Filter(const II_NumericList *nl, double min, double max, int min_inclusive, int max_inclusive);
void II_NumericList_Free(II_NumericList *nl);
/* From already-decoded host arrays (freqs may be NULL = all 1).  docIds strictly ascending. */
II_PostingList *II_PostingList_FromArrays(const uint64_t *doc_ids, const uint32_t *freqs, size_t n);
/* Adopt COPIES of device arrays (docIds u32 ascending, freqs u32). */
II_PostingList *II_PostingList_FromDevice(const uint32_t *d_doc_ids, const uint32_t *d_freqs, size_t n);
size_t II_PostingList_Len(const II_PostingList *pl);
size_t II_PostingList_NumEstimated(const II_PostingList *pl); /* InvIndIterator::num_estimated = unique_docs */
void II_PostingList_Free(II_PostingList *pl);

/* ---- per-document metadata the scorers read (RSDocumentMetadata: score, docLen, maxTermFreq) ---- */
typedef struct II_DocTable II_DocTable;
/* Arrays are indexed by docId (entry 0 unused); any of them may be NULL (docLen defaults to 0,
 * score to 1.0f, maxFreq to 1). */
II_DocTable *II_DocTable_New(size_t max_doc_id, const uint32_t *doc_len, const float *doc_score,
                             const uint32_t *max_term_freq);
/* Same from device arrays (copied). */
II_DocTable *II_DocTable_FromDevice(size_t max_doc_id, const uint32_t *d_doc_len, const float *d_doc_score,
                                    const uint32_t *d_max_term_freq);
void II_DocTable_Free(II_DocTable *dt);
/* Document payloads (dmd->payload, src/redisearch.h RSDocumentMetadata) for the HAMMING scorer: the bytes of docId d are
 * payloads[offsets[d] .. offsets[d + 1]), offsets has max_doc_id + 2 entries; an empty range = the document has no payload. */
int II_DocTable_SetPayloads(II_DocTable *dt, const uint8_t *payloads, const uint64_t *offsets);

/* ---- iterator algebra on device ---------------------------------------------------------------- */
typedef struct II_ResultSet II_ResultSet;

/* AND of n (1..32) posting lists: ascending docIds present in all of them — Intersection::read
 * (RS/rqe_iterators/src/intersection.rs:428-452) run to EOF.  Children are ordered by
 * num_estimated ascending, stable, exactly like Intersection::new (:103-169); per-hit child freqs
 * are kept in that order for the scorers. */
II_ResultSet *II_Intersect(II_PostingList *const *lists, size_t n);
/* OR of n (1..1024) posting lists run to EOF — a prefix / fuzzy expansion is a union of up to MAXEXPANSIONS (200) terms.
 * Up to min_union_iter_heap = 20 children the reference uses UnionFlat (RS/rqe_iterators/src/union_flat.rs:324-348): the per-hit
 * children come back in ITS aggregate order (the active array after swap_remove_child :174-180), so scores are bit-equal.  Above
 * 20 it uses UnionHeap (union_heap.rs), whose aggregate order follows the heap array: same docIds, same children per docId, the
 * scorer's sum is taken in list order here (last-bit differences possible).  quick_exit != 0 keeps docIds only (quick mode
 * reports a single child, union_flat.rs:433-524). */
II_ResultSet *II_Union(II_PostingList *const *lists, size_t n, int quick_exit);
/* nq independent ANDs in one call (e.g. the pre-filters of a batch of hybrid queries): all of them are enqueued, each on its own
 * stream, before anything is waited for.  out[i] = the result set of lists[i][0 .. n_lists[i]) or NULL; returns how many were built. */
size_t II_IntersectBatch(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, II_ResultSet **out);
/* AND with NOT / OPTIONAL children — the "a -b" / "a ~b" query shapes (RS/rqe_iterators/src/not.rs, optional.rs as children of
 * an Intersection): modes[i] 0 = required, 1 = NOT (docIds of lists[i] are excluded), 2 = OPTIONAL (never rejects; where
 * the docId is present its freq is kept).  Excluded / absent children yield the reference's virtual results: freq 0, no
 * contribution to any scorer (src/ext/default.c:289-297).  At least one child must be required. */
II_ResultSet *II_IntersectEx(II_PostingList *const *lists, const int *modes, size_t n);
/* AND under the reference's proximity constraints — exact phrases and "within N words" (Intersection::relevancy check,
 * RS/rqe_iterators/src/intersection.rs:201-242, -> RSIndexResult::is_within_range, RS/index_result/src/core/proximity.rs:
 * within_range_in_order :127-180, within_range_unordered :184-220, is_within_range :262-299).  max_slop < 0 = no limit;
 * in_order != 0 = the terms must appear in the order of `lists`, which is then also the aggregate child order (the reference
 * does not sort the children of an in-order intersection, intersection.rs:143).  One thread per candidate hit walks the term
 * positions of its children on the device; hits out of range are dropped, order and per-child freqs are kept.  modes may be
 * NULL; NOT children and absent OPTIONAL children are virtual results without positions and are left out of the check, as
 * in the reference.  Every other list must come from II_PostingList_FromBlocksBatchOffsets; n <= 8. */
II_ResultSet *II_IntersectPhrase(II_PostingList *const *lists, const int *modes, size_t n, int32_t max_slop, int in_order);
size_t II_ResultSet_Len(const II_ResultSet *rs);
void II_ResultSet_Free(II_ResultSet *rs);
/* The same nq ANDs with no host wait at all: each is enqueued on one of the library's streams and `stream` (a cudaStream_t cast
 * to void*, NULL = the legacy default stream) is made to wait, through events, for every one of them.  out[i] = a result set whose
 * length is still pending on the device, or NULL (an empty child, no list or more than 32 lists: the caller passes cap 0 for it);
 * returns how many were built.  Its docIds (II_ResultSet_DeviceDocIds) and u32 count (II_ResultSet_DeviceLen) are valid in
 * `stream` order; II_ResultSet_Capacity is the host bound on the count (the shortest list's length).  Every other accessor (Len,
 * Fetch, TopN, Score, the iterators, ...) first waits for the set and then behaves as on a set from II_IntersectBatch. */
size_t II_IntersectBatchDevice(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, void *stream, II_ResultSet **out);
const uint32_t *II_ResultSet_DeviceLen(const II_ResultSet *rs); /* u32 hit count, valid in stream order */
size_t II_ResultSet_Capacity(const II_ResultSet *rs);           /* host upper bound on the count */
/* Free rs once the work enqueued on `stream` so far is done, without waiting: the library's stream waits for an event recorded
 * on `stream` before the memory goes back to the pool.  II_ResultSet_Free releases the memory in the library's own stream order,
 * so kernels of the caller's stream still reading the docIds would see it handed out again; use this after enqueuing a consumer
 * on another stream. */
void II_ResultSet_FreeAfter(II_ResultSet *rs, void *stream);
/* nq ORs with no host wait: out[i] = II_Union(lists[i], n_lists[i], quick_exit) as a set whose count is pending on the device, or
 * NULL when query i has no list or all its lists are empty.  Once settled (any host accessor: Len, Fetch, TopN, Score, ChildOrder,
 * IntoChild, the result iterator) every set is indistinguishable from II_Union's: docIds, count, per-hit child freq rows, aggregate
 * child order, num_estimated, cap.  II_ResultSet_DeviceDocIds / DeviceLen / Capacity are valid in `stream` order as for
 * II_IntersectBatchDevice, and `stream` waits, through an event, for everything the call enqueued.  The whole batch takes 4
 * launches (quick_exit) or 6, whatever nq and the number of lists; nothing reads a count back.  Returns 0, or -1 before anything is
 * enqueued (a query with more than 1024 lists, a NULL list, or a list carrying a nested set, II_ResultSet_IntoChild);
 * *built (may be NULL) = the sets created. */
int II_UnionBatchDevice(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, int quick_exit, void *stream,
                        II_ResultSet **out, size_t *built);
typedef struct {
    double min, max;
    int min_inclusive, max_inclusive;
} II_NumericRange;
/* nq numeric range filters with no host wait.  Query i: the leaves the host's range-tree walk picked for its filter, and the
 * filter.  out[i] = the ascending docIds, one per document, of the documents with at least one value in the range in any of
 * those leaves (NumericFilter::value_in_range, bit for bit) — the set II_Union(quick) over II_NumericList_Filter of each leaf
 * builds (freq 1, docIds only, num_estimated = the sum of the filtered leaves' lengths once settled) — pending as above, or NULL
 * when the query has no leaf record at all.  No intermediate list per leaf: the range test runs in the union's mark pass.
 * 4 launches per batch.  Returns 0, or -1 before anything is enqueued (more than 1024 leaves, a NULL leaf or no ranges). */
int II_NumericFilterBatchDevice(size_t nq, II_NumericList *const *const *leaves, const size_t *n_leaves, const II_NumericRange *ranges,
                                void *stream, II_ResultSet **out, size_t *built);
/* One child of a filter-mode AND: a posting list, or a set of II_IntersectBatchDevice / II_UnionBatchDevice /
 * II_NumericFilterBatchDevice / II_IntersectFilterBatchDevice (or any other set), pending or settled.  Both NULL: an empty child
 * (the NULL those calls hand out for a filter that matches nothing). */
typedef struct {
    const II_PostingList *list;
    const II_ResultSet *set;
    int mode; /* 0 required, 1 NOT */
} II_FilterChild;
/* nq ANDs of lists and sets in FILTER MODE with no host wait — `@brand:nike @category:{shoes|boots}`, `@brand:nike
 * @price:[50 200]`, `@category:{shoes|boots} @price:[50 200] -@tag:{sale}` ahead of a KNN — without settling the ORs and ranges
 * first.  out[q] = the ascending docIds and count of the AND of children[q][0 .. n_children[q]), each set counting as the docIds
 * it holds once settled: what II_IntersectEx gives over the same lists plus II_PostingList_FromDevice of each set's docIds, with
 * the same modes.  out[q] is NULL when a required child is empty on the host (a list of length 0, a set of capacity 0, an empty
 * child); an empty NOT child excludes nothing.
 * Filter mode: a set carries docIds, count, num_estimated and the child order, no per-child freq rows (has no scores): II_Score
 * returns -1 and II_ResultSet_IntoChild NULL, as for quick unions.  Its shape: n_children = n_children[q]; capacity = the
 * smallest host bound of a required child (a list's length, a set's II_ResultSet_Capacity); num_estimated = the smallest of the
 * required children's, a set counting with its own num_estimated and sort weight as II_ResultSet_IntoChild would give them (1
 * for an OR, 1 / its children for an AND); child order = Intersection::new's stable sort by num_estimated x sort weight, NOT
 * children last.  Where a required child's estimate is still on the device (a pending numeric set, or a pending set of this call
 * that has one), the order and the estimate are worked out when the set settles; II_ResultSet_ChildOrder then settles it first.
 * II_ResultSet_DeviceDocIds / DeviceLen / Capacity are valid in `stream` order; DeviceLen[1] holds the set's num_estimated and
 * DeviceLen[2 + i] child i's (both saturated at 2^32 - 1).  An output is a valid set child of a later call and a valid KNN
 * filter (VecSimB200_TopKFilteredBatchDevice).
 * No host wait: the library's stream waits for each pending child set's own kernels through events, the tables go up from
 * pinned staging, nothing reads a count back, and `stream` waits for the batch through an event.  3 launches per batch, whatever
 * nq and the number of children.  The inputs are borrowed: a child set may be freed (II_ResultSet_Free / FreeAfter) right after
 * the call, from any thread; its memory is released once the call's kernels are done with it.  One set may be a child of calls
 * on several threads at once.
 * Returns 0, or -1 before anything is enqueued: NULL arguments, a query with more than 32 children or no required child, a mode
 * other than 0 or 1, a child with both `list` and `set`.  *built (may be NULL) = the sets created. */
int II_IntersectFilterBatchDevice(size_t nq, const II_FilterChild *const *children, const size_t *n_children, void *stream,
                                  II_ResultSet **out, size_t *built);
/* nq ORs of lists and sets in FILTER MODE with no host wait — `(@brand:nike @color:red) | (@brand:adidas @color:blue)`,
 * `@price:[0 50] | @price:[500 +inf]`, `(@category:{shoes} @price:[50 200]) | @brand:nike` ahead of a KNN — without settling the
 * ANDs and ranges first.  out[q] = the ascending docIds and count of the OR of children[q][0 .. n_children[q]), each set counting
 * as the docIds it holds once settled: what II_Union(quick_exit = 1) gives over the same lists plus II_PostingList_FromDevice of
 * each set's docIds.  out[q] is NULL when every child is empty on the host (a list of length 0, a set of capacity 0, both NULL).
 * Filter mode as for II_IntersectFilterBatchDevice: docIds, count, num_estimated and the child order, no per-child freq rows;
 * II_Score returns -1 and II_ResultSet_IntoChild NULL, as for quick unions.  Its shape is the one II_Union gives a quick union:
 * n_children = n_children[q]; the child order is the identity; child tags: a list keeps its own, an OR or numeric set is 1, an
 * AND set 2, an empty child 4; num_estimated = the sum of the children's (a set counting with its own); capacity = min(the sum of
 * the children's host bounds (a list's length, a set's II_ResultSet_Capacity), the highest docId the children can hold + 1).
 * Where a child's estimate is still on the device (a pending numeric set, or a pending filter-mode set that has one) the sum is
 * formed there and worked out when the set settles.  DeviceLen[1] holds num_estimated, saturated at 2^32 - 1.
 * II_ResultSet_DeviceDocIds / DeviceLen / Capacity are valid in `stream` order.  An output is a valid set child of a later call
 * of this function or of II_IntersectFilterBatchDevice, and a valid KNN filter (VecSimB200_TopKFilteredBatchDevice).
 * No host wait, and the inputs are borrowed, as for II_IntersectFilterBatchDevice.  4 launches per batch (plus one clear and one
 * upload), whatever nq and the number of children.  Every set carries host-known bounds on its docIds, which size the bitmap
 * window of each query.
 * Returns 0, or -1 before anything is enqueued: NULL arguments, a query with more than 1024 children, a mode other than 0 (no
 * NOT under an OR), a child with both `list` and `set`, a list carrying a nested set (II_ResultSet_IntoChild).  *built (may be
 * NULL) = the sets created. */
int II_UnionFilterBatchDevice(size_t nq, const II_FilterChild *const *children, const size_t *n_children, void *stream,
                              II_ResultSet **out, size_t *built);

/* ---- scoring ------------------------------------------------------------------------------------ */
typedef enum {
    II_SCORER_BM25STD = 0,      /* default scorer; src/ext/default.c:241-316 */
    II_SCORER_BM25 = 1,         /* legacy; :164-233, divided by GetSlop = IndexResult_MinOffsetDelta (src/index_result/index_result.c:51-108)
                                 * over the term positions of the hit when the lists carry them, else `children - 1` as the reference */
    II_SCORER_TFIDF = 2,        /* :68-146 (same slop factor) */
    II_SCORER_TFIDF_DOCNORM = 3,/* :148-153 */
    II_SCORER_DOCSCORE = 4,     /* :366-371 */
    II_SCORER_BM25STD_TANH = 5, /* :339-359 */
    II_SCORER_DISMAX = 6,       /* :378-461 */
    II_SCORER_HAMMING = 7       /* :475-497: needs the payloads (II_DocTable_SetPayloads) and goes through II_ScoreHamming */
} II_Scorer;

/* Per query term, in the ORIGINAL order of the `lists` argument. */
typedef struct {
    double weight;   /* leaf result weight (query node weight, default 1.0) */
    double idf;      /* QueryTerm_GetIDF      — II_CalculateIDF      */
    double bm25_idf; /* QueryTerm_GetBM25_IDF — II_CalculateIDF_BM25 */
} II_TermParams;

double II_CalculateIDF(size_t total_docs, size_t term_docs);      /* RS/idf/src/lib.rs:67 */
double II_CalculateIDF_BM25(size_t total_docs, size_t term_docs); /* RS/idf/src/lib.rs:103 */

/* NESTED aggregates: an evaluated AND / OR becomes ONE child of another aggregate — `(a|b) c`, the expansions of a stemmed term
 * under an AND, a phrase inside a larger query.  Returns the list view of its hits (docIds; freq = the sum of its children's,
 * like RSAggregateResult) that II_Intersect* / II_Union accept; the view carries the set, so that
 *   - the scorers recurse into it: weight * sum (DISMAX over a union: max) over ITS children
 *     (src/ext/default.c:75-95 tfidfRecursive, :183-199 bm25Recursive, :272-289 bm25StdRecursive, :393-438 dismaxRecursive);
 *   - the proximity checks and GetSlop see the k-way merge of its children's term positions, duplicates kept
 *     (src/offset_vector.c:100-140,216-239; RS/index_result/src/core/proximity.rs:53-67), and it COUNTS as having offsets by
 *     the kind mask of its children (src/index_result/index_result.c:23-35) whatever the streams hold.
 * CONSUMES rs (also on failure: NULL).  terms: of rs's children in the order they were given to its constructor; weight: the
 * nested node's own; the parent's II_TermParams entry for this child is not read.  with_positions != 0 builds the merged
 * positions now (a parent with slop / in-order needs them up front; GetSlop builds them on demand).  Quick unions (no per-child
 * freqs) cannot be nested this way. */
II_PostingList *II_ResultSet_IntoChild(II_ResultSet *rs, const II_TermParams *terms, double weight, int with_positions);
/* Score every hit of `rs` on device.  agg_weight = weight of the intersection/union node.
 * Returns 0, or -1 on failure. */
int II_Score(II_ResultSet *rs, II_Scorer scorer, const II_TermParams *terms, double agg_weight,
             const II_IndexStats *stats, const II_DocTable *docs, double min_score, uint64_t tanh_factor);

/* HAMMING scorer (src/ext/default.c:475-497) over every hit: 1 / (bit distance between the query payload and the document's
 * payload + 1); 0 for documents without a payload or of another length. */
int II_ScoreHamming(II_ResultSet *rs, const II_DocTable *docs, const void *qdata, size_t qdatalen);

/* Copy results to the host.  Any output pointer may be NULL.  child_freqs is [n_children][len]
 * (children in aggregate order; 0 = child absent, union only).  scores are 0 before II_Score. */
int II_ResultSet_Fetch(const II_ResultSet *rs, uint64_t *doc_ids, double *scores, uint32_t *child_freqs);
size_t II_ResultSet_NumChildren(const II_ResultSet *rs);
/* child_order[i] = index in the `lists` argument of aggregate child i (a set of II_IntersectFilterBatchDevice whose order waits
 * for estimates on the device is settled first). */
void II_ResultSet_ChildOrder(const II_ResultSet *rs, uint32_t *child_order);
/* Best `n` hits by (score desc, docId asc) — RPSorter's cmpByScore, src/result_processor.c:834-850 —
 * selected on device.  Returns the number written. */
size_t II_ResultSet_TopN(const II_ResultSet *rs, size_t n, uint64_t *doc_ids, double *scores);
/* Device views (valid until the result set is freed): docIds u32[len], scores f64[len]. */
const uint32_t *II_ResultSet_DeviceDocIds(const II_ResultSet *rs);
const double *II_ResultSet_DeviceScores(const II_ResultSet *rs);

/* One call for the common query: AND (or OR) of term lists, score, top-N; host arrays out.
 * Thread-safe: every calling thread owns a stream inside the library (one iterator tree per RediSearch worker
 * thread, src/util/workers.c), so concurrent searches over shared posting lists overlap on the device.
 * II_GetStats reports the calling thread's counters. */
size_t II_SearchTopN(II_PostingList *const *lists, size_t n, int is_union, II_Scorer scorer,
                     const II_TermParams *terms, double agg_weight, const II_IndexStats *stats,
                     const II_DocTable *docs, size_t top_n, uint64_t *doc_ids, double *scores, size_t *total_hits);
/* `nq` independent searches in one call (the dispatch shim batches concurrent FT.SEARCHes the way
 * VecSimB200_TopKQueryBatch batches KNN queries).  lists[i] / n_lists[i] / terms[i] describe query i; outputs are
 * [nq][top_n] row-major, counts[i] = hits written for query i, total_hits[i] (optional) = size of its AND/OR.
 * The queries are spread over a pool of 8 streams inside the library.  top_n <= 1024.  Returns 0, or -1 on a bad
 * argument / missing device. */
int II_SearchTopNBatch(size_t nq, II_PostingList *const *const *lists, const size_t *n_lists, int is_union, II_Scorer scorer,
                       const II_TermParams *const *terms, double agg_weight, const II_IndexStats *stats, const II_DocTable *docs,
                       size_t top_n, uint64_t *doc_ids, double *scores, size_t *counts, size_t *total_hits);

/* Multi-GPU: postings are sharded by docId range with the same boundaries as the vector rows (SURVEY.md §8e); every
 * shard runs II_SearchTopN on its slice with the GLOBAL statistics (numDocs, avgDocLen, per-term idf), and the
 * coordinator merges the per-shard lists — what src/module.c:3139-3176 does with per-shard replies.  scores / doc_ids
 * are [num_shards][per_shard], counts[g] entries valid; writes the best n by (score desc, docId asc), returns how many. */
size_t II_MergeShardTopN(const double *scores, const uint64_t *doc_ids, const size_t *counts, size_t num_shards, size_t per_shard,
                         size_t n, uint64_t *out_ids, double *out_scores);

/* ---- term -> device posting list cache ------------------------------------------------------------------------------
 * Hot terms stay decoded in HBM between queries; the host decode / H2D leaves the query path (SURVEY.md §8f1).
 * keys[i] identifies a term's inverted index (e.g. the InvertedIndex pointer), versions[i] must change whenever that index
 * is written or garbage-collected — e.g. (gc_marker << 32) | num_entries: the gc_marker is what the reference's readers
 * compare in needs_revalidation (RS/inverted_index/src/reader/core.rs:372-374, bumped by the GC at index/core.rs:436), the
 * entry count moves with every append.  Acquire returns resident lists for (key, version) hits WITHOUT touching the blocks
 * and decodes all misses together in one II_PostingList_FromBlocksBatch; a stale version is dropped and rebuilt.  The
 * returned handles are pinned (never evicted, never freed) until II_TermCache_Release; they must not be passed to
 * II_PostingList_Free.  Eviction is LRU over unpinned lists once resident_bytes exceeds max_device_bytes.  Thread-safe. */
typedef struct II_TermCache II_TermCache;
typedef struct {
    size_t hits, misses, evictions, resident_bytes, resident_lists;
} II_TermCacheStats;
II_TermCache *II_TermCache_New(size_t max_device_bytes);
void II_TermCache_Free(II_TermCache *cache);
/* Returns how many of the n lists are available in out[] (NULL = could not be built). */
size_t II_TermCache_Acquire(II_TermCache *cache, size_t n, const uint64_t *keys, const uint64_t *versions,
                            const II_BlockView *const *blocks, const size_t *nblocks, II_Codec codec, II_PostingList **out);
void II_TermCache_Release(II_TermCache *cache, size_t n, II_PostingList *const *lists);
void II_TermCache_Invalidate(II_TermCache *cache, uint64_t key); /* from the index writer / GC, when it is cheaper than versions */
/* on: lists decoded from now on keep their term positions (any codec that stores them: Full, FreqsOffsets, OffsetsOnly, FieldsOffsets and the wide variants) so that phrase / slop intersections can use them */
void II_TermCache_KeepOffsets(II_TermCache *cache, int on);
II_TermCacheStats II_TermCache_GetStats(II_TermCache *cache);

/* ---- QueryIterator facade ------------------------------------------------------------------------ */
/* Takes ownership of `rs` (downloads docIds/scores once).  Free through it->Free(it). */
II_QueryIterator *II_NewResultIterator(II_ResultSet *rs, double weight);

/* ---- the reference's constructors and scorer extension on top of the device algebra ------------------------------------
 * NewIntersectionIterator / NewUnionIterator carry the reference's exact signatures (RS/headers/iterators_ffi.h:309,594;
 * `QueryIterator` == II_QueryIterator, layout-identical) and ownership rules: they take over the `its` array (freed with
 * RedisModule_Free when the host exports it, else free) and every child.  Children may be device iterators (term leaves,
 * NOT / OPTIONAL wrappers, nested results: they stay on the device) or FOREIGN iterators of the host (numeric, tag, geo ...
 * leaves: drained once through Read() and uploaded).  The reduction rules of intersection.rs:363-417 / union_reducer.rs:30-66
 * are applied (no children -> empty, NULL / empty child, wildcard stripping, single survivor returned as is).  The tree is
 * evaluated on the device at construction; the returned iterator walks the finished result set.  Phrase constraints
 * (max_slop >= 0, in_order) are evaluated on the device (II_IntersectPhrase) when every child is a device term leaf carrying
 * its term positions and there are at most 8 of them; otherwise NULL is returned with nothing consumed and the caller keeps
 * the reference's iterator for that node. */
II_QueryIterator *NewIntersectionIterator(II_QueryIterator **its, size_t num, int32_t max_slop, bool in_order, double weight);
II_QueryIterator *NewUnionIterator(II_QueryIterator **its, int32_t num, bool quick_exit, double weight, int /* QueryNodeType */ type_,
                                   const char *q_str, const void /* IteratorsConfig */ *config);
/* The term leaf under the reference's own name and signature (RS/headers/iterators_ffi.h:404; Term::new,
 * RS/rqe_iterators/src/inverted_index/term.rs:77-100).  Everything it needs from the host is resolved with dlsym in the host
 * process: InvertedIndex_Flags / _NumDocs and the block accessors (inverted_index_ffi.h), IndexSpec_GetStats (src/spec.h:509),
 * QueryTerm_SetIDFs / Term_Free (query_term_ffi.h:108,119); `sctx` is read as {redisCtx, spec, ...} (src/search_ctx.h:60-64).
 * Decoded lists go through the cache set with II_SetDefaultTermCache (NULL: decoded per iterator).  Returns NULL with nothing
 * consumed when an accessor is missing or the index is not a term index: the caller keeps the reference's iterator. */
typedef struct {
    uint8_t tag; /* 0 = Index (field index, used for expiration checks only), 1 = Mask — RS/headers/field.h:29-57 */
    unsigned __int128 mask __attribute__((aligned(16)));
} II_FieldMaskOrIndex;
II_QueryIterator *NewInvIndIterator_TermQuery(const void *idx, const void *sctx, II_FieldMaskOrIndex field_mask_or_index, void *term,
                                              double weight);
void II_SetDefaultTermCache(II_TermCache *cache);
/* DocIdsOnly indexes: 1 = the host runs with raw docId encoding (RawDocIdsOnly), which the index flags do not say */
void II_SetRawDocIdEncoding(int raw);
/* IndexFlags (src/spec.h:171-181) -> II_Codec, the table of NewInvertedIndex_Ex (inverted_index_ffi/src/lib.rs:49-165); -1 = not a
 * term index */
int II_CodecFromIndexFlags(uint32_t flags, int raw_doc_id_encoding);
II_QueryIterator *II_NewEmptyIterator(void);
/* rqe_iterators/src/wildcard.rs:83-180: every docId 1..top_id as a virtual result (freq 1, all fields) of the given weight; the
 * second name is the reference's (RS/headers/iterators_ffi.h:647).  Stripped by our AND, taken over by a quick OR
 * (union_reducer.rs:41-53), a device list 1..top_id inside a full OR. */
II_QueryIterator *II_NewWildcardIterator(t_docId top_id, double weight);
II_QueryIterator *NewWildcardIterator_NonOptimized(t_docId max_id, double weight);
/* Term leaf over a device posting list (what NewInvIndIterator_TermQuery, iterators_ffi.h:404, yields): weight = the query
 * node's weight, idf / bm25_idf = QueryTerm_GetIDF / QueryTerm_GetBM25_IDF of the term. */
II_QueryIterator *II_NewTermIterator(II_PostingList *pl, int take_ownership, double weight, double idf, double bm25_idf);
/* The same straight from the host's InvertedIndex*: its block accessors (inverted_index_ffi.h:102-132,286,387,425,444, plus
 * IndexBlock_DataLen — INTEGRATION.md §2) are resolved in the host process with dlsym.  With a cache the decoded list is
 * shared across queries, keyed by the index pointer and versioned by (gc_marker, num_entries). */
II_QueryIterator *II_NewTermIterator_FromIndex(const void *inverted_index, II_Codec codec, double weight, double idf, double bm25_idf,
                                               II_TermCache *cache);
/* NOT / OPTIONAL over a device term leaf (iterators_ffi.h NewNotIterator / NewOptionalIterator without the QueryEvalCtx): as a
 * child of NewIntersectionIterator they fuse into the membership kernel (exclusion / optional contribution). */
II_QueryIterator *II_NewNotIterator(II_QueryIterator *child, t_docId max_doc_id, double weight);
II_QueryIterator *II_NewOptionalIterator(II_QueryIterator *child, t_docId max_doc_id, double weight);
/* Per-document metadata the *.B200 scorers read (one table per index spec; the default applies to iterators built afterwards). */
void II_SetDefaultDocTable(const II_DocTable *docs);
/* Scorer extension entry point: `redis-server --loadmodule redisearch.so EXTLOAD libii_b200.so` makes Extension_LoadDynamic
 * (src/extension.c:121-145) dlsym this symbol; it registers BM25STD.B200, BM25.B200, TFIDF.B200, TFIDF.DOCNORM.B200,
 * DOCSCORE.B200, BM25STD.TANH.B200 and DISMAX.B200 through ctx->RegisterScoringFunction (RSExtensionCtx, src/redisearch.h:282).
 * Each is an RSScoringFunction (src/redisearch.h:277): called per result with the iterator's `current`, it scores the WHOLE
 * result set on the device at the first call and returns the stored value afterwards. */
int RS_ExtensionInit(void *rs_extension_ctx);

/* ---- statistics for bench / roofline ---------------------------------------------------------------- */
typedef struct {
    uint64_t kernel_launches;
    double intersect_device_us; /* CUDA-event time of the last II_Intersect / II_Union kernels */
    double score_device_us;     /* ... of the last II_Score */
    double decode_host_us;      /* host decode wall time of the last II_PostingList_FromBlocks */
    double h2d_us;
} II_Stats;
II_Stats II_GetStats(bool reset);
/* EXPLAINSCORE of ONE result given as a flattened result tree (node 0 the root, parent[i] < i, children in index order; kind 0 term,
 * 1 intersection, 2 union, 3 virtual, 4 numeric; term_str: the text printed for term leaves, may be NULL): the explanation tree the
 * reference's scorer builds with its EXPLAIN macro (src/ext/default.c:68-497, strExpCreateParent :58-65), serialised one node per
 * line as "<depth> <string>\n" in pre-order; *score_out = the score.  Host code, no device.  Returns the bytes needed (excluding NUL).
 * The *.B200 scorers use the same builder when ScoringFunctionArgs.scrExp is set (INTEGRATION.md section 2). */
size_t II_ExplainTree(int scorer, size_t n_nodes, const int32_t *parent, const int32_t *kind, const uint32_t *freq, const double *weight,
                      const double *idf, const double *bm25_idf, const char *term_str, uint32_t doc_len, uint32_t max_freq, float doc_score,
                      double avg_doc_len, int slop, double min_score, uint64_t tanh_factor, double *score_out, char *buf, size_t cap);
const char *II_Version(void);

#ifdef __cplusplus
}
#endif
#endif /* II_B200_H */
