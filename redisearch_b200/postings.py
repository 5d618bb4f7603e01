"""ctypes face of libii_b200.so (include/ii_b200.h): posting lists in HBM, AND / OR on device, the
reference's scorers, top-N and the QueryIterator facade.  No compute happens here."""
import ctypes as C

import numpy as np

from ._lib import load_library

CODEC_FULL, CODEC_FREQS_ONLY, CODEC_FREQS_FIELDS, CODEC_FIELDS_ONLY, CODEC_DOCIDS_ONLY, CODEC_RAW_DOCIDS_ONLY = range(6)
SCORER_BM25STD, SCORER_BM25, SCORER_TFIDF, SCORER_TFIDF_DOCNORM, SCORER_DOCSCORE, SCORER_BM25STD_TANH, SCORER_DISMAX = range(7)
ITERATOR_OK, ITERATOR_NOTFOUND, ITERATOR_EOF, ITERATOR_TIMEOUT = range(4)


class II_BlockView(C.Structure):
    _fields_ = [("first_doc_id", C.c_uint64), ("last_doc_id", C.c_uint64), ("num_entries", C.c_uint16),
                ("data", C.POINTER(C.c_uint8)), ("len", C.c_size_t)]


class II_TermParams(C.Structure):
    _fields_ = [("weight", C.c_double), ("idf", C.c_double), ("bm25_idf", C.c_double)]


class II_IndexStats(C.Structure):
    _fields_ = [("numDocs", C.c_size_t), ("numTerms", C.c_size_t), ("avgDocLen", C.c_double)]


class II_NumericRange(C.Structure):
    _fields_ = [("min", C.c_double), ("max", C.c_double), ("min_inclusive", C.c_int), ("max_inclusive", C.c_int)]


class II_FilterChild(C.Structure):
    _fields_ = [("list", C.c_void_p), ("set", C.c_void_p), ("mode", C.c_int)]


class II_Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("intersect_device_us", C.c_double), ("score_device_us", C.c_double),
                ("decode_host_us", C.c_double), ("h2d_us", C.c_double)]


class II_TermCacheStats(C.Structure):
    _fields_ = [("hits", C.c_size_t), ("misses", C.c_size_t), ("evictions", C.c_size_t), ("resident_bytes", C.c_size_t),
                ("resident_lists", C.c_size_t)]


class _ResultData(C.Structure):
    _fields_ = [("tag", C.c_uint8), ("_pad", C.c_uint8 * 7), ("metric", C.c_double), ("_rest", C.c_uint8 * 24)]


class II_IndexResult(C.Structure):
    _fields_ = [("docId", C.c_uint64), ("dmd", C.c_void_p), ("fieldMask_lo", C.c_uint64), ("fieldMask_hi", C.c_uint64),
                ("freq", C.c_uint32), ("data", _ResultData), ("metrics", C.c_void_p), ("weight", C.c_double),
                ("hasFieldExpiration", C.c_bool)]


class II_QueryIterator(C.Structure):
    pass


_QI = C.POINTER(II_QueryIterator)
II_QueryIterator._fields_ = [
    ("type", C.c_uint32), ("atEOF", C.c_bool), ("lastDocId", C.c_uint64), ("current", C.POINTER(II_IndexResult)),
    ("NumEstimated", C.CFUNCTYPE(C.c_size_t, _QI)), ("Read", C.CFUNCTYPE(C.c_int, _QI)),
    ("SkipTo", C.CFUNCTYPE(C.c_int, _QI, C.c_uint64)), ("Revalidate", C.CFUNCTYPE(C.c_int, _QI, C.c_void_p)),
    ("Free", C.CFUNCTYPE(None, _QI)), ("Rewind", C.CFUNCTYPE(None, _QI)), ("ProfileChildren", C.c_void_p),
    ("PrintProfile", C.c_void_p)]

_P, _SZ = C.c_void_p, C.c_size_t
SIGNATURES = [
    ("II_PostingList_FromBlocks", _P, [C.POINTER(II_BlockView), _SZ, C.c_int, C.c_uint32, C.c_int]),
    ("II_PostingList_FromBlocksBatch", _SZ, [_SZ, _P, _P, C.c_int, _P]),
    ("II_PostingList_FromBlocksBatchOffsets", _SZ, [_SZ, _P, _P, C.c_int, _P]),
    ("II_PostingList_HasOffsets", C.c_int, [_P]),
    ("II_PostingList_FromArrays", _P, [_P, _P, _SZ]),
    ("II_PostingList_FromDevice", _P, [_P, _P, _SZ]),
    ("II_PostingList_Len", _SZ, [_P]),
    ("II_PostingList_NumEstimated", _SZ, [_P]),
    ("II_PostingList_Free", None, [_P]),
    ("II_DocTable_New", _P, [_SZ, _P, _P, _P]),
    ("II_DocTable_FromDevice", _P, [_SZ, _P, _P, _P]),
    ("II_DocTable_Free", None, [_P]),
    ("II_Intersect", _P, [_P, _SZ]),
    ("II_Union", _P, [_P, _SZ, C.c_int]),
    ("II_ResultSet_Len", _SZ, [_P]),
    ("II_ResultSet_Free", None, [_P]),
    ("II_ExplainTree", C.c_size_t, [C.c_int, C.c_size_t, _P, _P, _P, _P, _P, _P, C.c_char_p, C.c_uint32, C.c_uint32, C.c_float, C.c_double,
                        C.c_int, C.c_double, C.c_uint64, _P, _P, C.c_size_t]),
    ("II_ResultSet_IntoChild", _P, [_P, _P, C.c_double, C.c_int]),
    ("II_CalculateIDF", C.c_double, [_SZ, _SZ]),
    ("II_CalculateIDF_BM25", C.c_double, [_SZ, _SZ]),
    ("II_ScoreHamming", C.c_int, [_P, _P, _P, _SZ]),
    ("II_DocTable_SetPayloads", C.c_int, [_P, _P, _P]),
    ("II_Score", C.c_int, [_P, C.c_int, C.POINTER(II_TermParams), C.c_double, C.POINTER(II_IndexStats), _P, C.c_double, C.c_uint64]),
    ("II_ResultSet_Fetch", C.c_int, [_P, _P, _P, _P]),
    ("II_ResultSet_NumChildren", _SZ, [_P]),
    ("II_ResultSet_ChildOrder", None, [_P, _P]),
    ("II_ResultSet_TopN", _SZ, [_P, _SZ, _P, _P]),
    ("II_ResultSet_DeviceDocIds", _P, [_P]),
    ("II_ResultSet_DeviceScores", _P, [_P]),
    ("II_SearchTopN", _SZ, [_P, _SZ, C.c_int, C.c_int, C.POINTER(II_TermParams), C.c_double, C.POINTER(II_IndexStats), _P, _SZ,
                            _P, _P, C.POINTER(_SZ)]),
    ("II_SearchTopNBatch", C.c_int, [_SZ, _P, _P, C.c_int, C.c_int, _P, C.c_double, C.POINTER(II_IndexStats), _P, _SZ, _P, _P, _P, _P]),
    ("II_MergeShardTopN", _SZ, [_P, _P, _P, _SZ, _SZ, _SZ, _P, _P]),
    ("II_NewResultIterator", _QI, [_P, C.c_double]),
    ("II_IntersectEx", _P, [_P, _P, _SZ]),
    ("II_IntersectBatch", _SZ, [_SZ, _P, _P, _P]),
    ("II_IntersectBatchDevice", _SZ, [_SZ, _P, _P, _P, _P]),
    ("II_ResultSet_DeviceLen", _P, [_P]),
    ("II_ResultSet_Capacity", _SZ, [_P]),
    ("II_ResultSet_FreeAfter", None, [_P, _P]),
    ("II_UnionBatchDevice", C.c_int, [_SZ, _P, _P, C.c_int, _P, _P, C.POINTER(_SZ)]),
    ("II_NumericFilterBatchDevice", C.c_int, [_SZ, _P, _P, _P, _P, _P, C.POINTER(_SZ)]),
    ("II_IntersectFilterBatchDevice", C.c_int, [_SZ, _P, _P, _P, _P, C.POINTER(_SZ)]),
    ("II_UnionFilterBatchDevice", C.c_int, [_SZ, _P, _P, _P, _P, C.POINTER(_SZ)]),
    ("II_IndexWriter_New", _P, [C.c_int]),
    ("II_IndexWriter_NewNumeric", _P, [C.c_int]),
    ("II_IndexWriter_Add", _SZ, [_P, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, _P, C.c_uint32]),
    ("II_IndexWriter_AddNumeric", _SZ, [_P, C.c_uint64, C.c_double]),
    ("II_IndexWriter_NumBlocks", _SZ, [_P]),
    ("II_IndexWriter_NumDocs", _SZ, [_P]),
    ("II_IndexWriter_Block", C.c_int, [_P, _SZ, C.POINTER(II_BlockView)]),
    ("II_IndexWriter_Free", None, [_P]),
    ("II_SetDefaultTermCache", None, [_P]),
    ("II_SetRawDocIdEncoding", None, [C.c_int]),
    ("II_CodecFromIndexFlags", C.c_int, [C.c_uint32, C.c_int]),
    ("II_NumericList_FromBlocks", _P, [C.POINTER(II_BlockView), _SZ]),
    ("II_NumericList_Len", _SZ, [_P]),
    ("II_NumericList_Fetch", C.c_int, [_P, _P, _P]),
    ("II_NumericList_Filter", _P, [_P, C.c_double, C.c_double, C.c_int, C.c_int]),
    ("II_NumericList_Free", None, [_P]),
    ("II_NewWildcardIterator", _QI, [C.c_uint64, C.c_double]),
    ("NewWildcardIterator_NonOptimized", _QI, [C.c_uint64, C.c_double]),
    ("II_PostingList_FromBlocksWideMask", _P, [_P, _SZ, C.c_int, _P, C.c_int]),
    ("II_IntersectPhrase", _P, [_P, _P, _SZ, C.c_int32, C.c_int]),
    ("NewIntersectionIterator", _QI, [_P, _SZ, C.c_int32, C.c_bool, C.c_double]),
    ("NewUnionIterator", _QI, [_P, C.c_int32, C.c_bool, C.c_double, C.c_int, C.c_char_p, _P]),
    ("II_NewEmptyIterator", _QI, []),
    ("II_NewTermIterator", _QI, [_P, C.c_int, C.c_double, C.c_double, C.c_double]),
    ("II_NewTermIterator_FromIndex", _QI, [_P, C.c_int, C.c_double, C.c_double, C.c_double, _P]),
    ("II_NewNotIterator", _QI, [_QI, C.c_uint64, C.c_double]),
    ("II_NewOptionalIterator", _QI, [_QI, C.c_uint64, C.c_double]),
    ("II_SetDefaultDocTable", None, [_P]),
    ("RS_ExtensionInit", C.c_int, [_P]),
    ("II_TermCache_New", _P, [_SZ]),
    ("II_TermCache_Free", None, [_P]),
    ("II_TermCache_Acquire", _SZ, [_P, _SZ, _P, _P, _P, _P, C.c_int, _P]),
    ("II_TermCache_Release", None, [_P, _SZ, _P]),
    ("II_TermCache_Invalidate", None, [_P, C.c_uint64]),
    ("II_TermCache_KeepOffsets", None, [_P, C.c_int]),
    ("II_TermCache_GetStats", II_TermCacheStats, [_P]),
    ("II_GetStats", II_Stats, [C.c_bool]),
    ("II_Version", C.c_char_p, []),
]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = load_library("libii_b200.so")
        for name, res, args in SIGNATURES:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class PostingList:
    def __init__(self, handle):
        if not handle:
            raise RuntimeError("posting list construction failed (no CUDA device, or unrepresentable docIds)")
        self.h = handle
        self.L = lib()

    @classmethod
    def from_arrays(cls, doc_ids, freqs=None):
        d = np.ascontiguousarray(doc_ids, dtype=np.uint64)
        f = np.ascontiguousarray(freqs, dtype=np.uint32) if freqs is not None else None
        return cls(lib().II_PostingList_FromArrays(_ptr(d), _ptr(f), len(d)))

    @classmethod
    def from_blocks(cls, blocks, codec, field_mask_filter=0, on_device=False):
        """blocks: list of (first_doc_id, last_doc_id, num_entries, bytes)."""
        arr = (II_BlockView * max(1, len(blocks)))()
        keep = []
        for i, (first, last, n, data) in enumerate(blocks):
            buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
            keep.append(buf)
            arr[i] = II_BlockView(first, last, n, C.cast(buf, C.POINTER(C.c_uint8)), len(data))
        if field_mask_filter >> 32:  # a u128 field-mask filter (the *Wide codecs)
            flt = (C.c_uint64 * 2)(field_mask_filter & 0xFFFFFFFFFFFFFFFF, field_mask_filter >> 64)
            return cls(lib().II_PostingList_FromBlocksWideMask(arr, len(blocks), codec, flt, int(on_device)))
        return cls(lib().II_PostingList_FromBlocks(arr, len(blocks), codec, field_mask_filter, int(on_device)))

    def __len__(self):
        return self.L.II_PostingList_Len(self.h)

    def num_estimated(self):
        return self.L.II_PostingList_NumEstimated(self.h)

    def close(self):
        if self.h:
            self.L.II_PostingList_Free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class IndexWriter:
    """II_IndexWriter: the reference's add_record on the host (byte-identical IndexBlocks)"""

    def __init__(self, codec=None, numeric=False, compress_floats=False):
        self.L = lib()
        self.h = self.L.II_IndexWriter_NewNumeric(int(compress_floats)) if numeric else self.L.II_IndexWriter_New(codec)
        if not self.h:
            raise RuntimeError("II_IndexWriter_New failed")

    def add(self, doc_id, freq=1, mask=1, offsets=b""):
        buf = (C.c_uint8 * max(1, len(offsets))).from_buffer_copy(offsets or b"\0")
        return self.L.II_IndexWriter_Add(self.h, doc_id, freq, mask & 0xFFFFFFFFFFFFFFFF, mask >> 64, buf, len(offsets))

    def add_numeric(self, doc_id, value):
        return self.L.II_IndexWriter_AddNumeric(self.h, doc_id, float(value))

    def num_docs(self):
        return self.L.II_IndexWriter_NumDocs(self.h)

    def blocks(self):
        out = []
        for i in range(self.L.II_IndexWriter_NumBlocks(self.h)):
            v = II_BlockView()
            assert self.L.II_IndexWriter_Block(self.h, i, C.byref(v)) == 0
            out.append((v.first_doc_id, v.last_doc_id, v.num_entries, bytes(C.cast(v.data, C.POINTER(C.c_uint8 * v.len)).contents) if v.len else b""))
        return out

    def __del__(self):
        try:
            if self.h:
                self.L.II_IndexWriter_Free(self.h)
                self.h = None
        except Exception:
            pass


class NumericList:
    """II_NumericList: a numeric index leaf decoded on the device"""

    def __init__(self, blocks):
        self.L = lib()
        arr = (II_BlockView * max(1, len(blocks)))()
        self._keep = []
        for i, (first, last, n, data) in enumerate(blocks):
            buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
            self._keep.append(buf)
            arr[i] = II_BlockView(first, last, n, C.cast(buf, C.POINTER(C.c_uint8)), len(data))
        self.h = self.L.II_NumericList_FromBlocks(arr, len(blocks))
        if not self.h:
            raise RuntimeError("II_NumericList_FromBlocks failed")

    def __len__(self):
        return self.L.II_NumericList_Len(self.h)

    def fetch(self):
        n = len(self)
        ids, vals = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.float64)
        if self.L.II_NumericList_Fetch(self.h, _ptr(ids), _ptr(vals)) != 0:
            raise RuntimeError("II_NumericList_Fetch failed")
        return ids, vals

    def filter(self, lo, hi, lo_inclusive=True, hi_inclusive=True):
        return PostingList(self.L.II_NumericList_Filter(self.h, lo, hi, int(lo_inclusive), int(hi_inclusive)))

    def __del__(self):
        try:
            if self.h:
                self.L.II_NumericList_Free(self.h)
                self.h = None
        except Exception:
            pass


class DocTable:
    def __init__(self, max_doc_id, doc_len=None, doc_score=None, max_term_freq=None):
        self.L = lib()
        dl = np.ascontiguousarray(doc_len, dtype=np.uint32) if doc_len is not None else None
        ds = np.ascontiguousarray(doc_score, dtype=np.float32) if doc_score is not None else None
        mf = np.ascontiguousarray(max_term_freq, dtype=np.uint32) if max_term_freq is not None else None
        self.h = self.L.II_DocTable_New(max_doc_id, _ptr(dl), _ptr(ds), _ptr(mf))
        if not self.h:
            raise RuntimeError("II_DocTable_New failed")

    def set_payloads(self, payloads):
        """payloads: list indexed by docId (0..max_doc_id) of bytes / None"""
        off = np.zeros(len(payloads) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(p) if p else 0 for p in payloads])
        blob = np.frombuffer(b"".join(p or b"" for p in payloads) or b"\0", dtype=np.uint8)
        if self.L.II_DocTable_SetPayloads(self.h, _ptr(blob), _ptr(off)) != 0:
            raise RuntimeError("II_DocTable_SetPayloads failed")

    def __del__(self):
        try:
            if self.h:
                self.L.II_DocTable_Free(self.h)
                self.h = None
        except Exception:
            pass


def _list_array(lists):
    return (C.c_void_p * len(lists))(*[pl.h for pl in lists])


class ResultSet:
    def __init__(self, handle):
        if not handle:
            raise RuntimeError("device iterator evaluation failed")
        self.h = handle
        self.L = lib()

    def __len__(self):
        return self.L.II_ResultSet_Len(self.h)

    def child_order(self):
        n = self.L.II_ResultSet_NumChildren(self.h)
        out = np.zeros(n, dtype=np.uint32)
        self.L.II_ResultSet_ChildOrder(self.h, _ptr(out))
        return out

    def score(self, scorer, terms, agg_weight, num_docs, avg_doc_len, doc_table=None, min_score=0.0, tanh_factor=4):
        """terms: list of (weight, idf, bm25_idf) in the ORIGINAL list order."""
        arr = (II_TermParams * len(terms))(*[II_TermParams(*t) for t in terms])
        st = II_IndexStats(num_docs, 0, avg_doc_len)
        rc = self.L.II_Score(self.h, scorer, arr, agg_weight, C.byref(st), doc_table.h if doc_table else None, min_score, tanh_factor)
        if rc != 0:
            raise RuntimeError("II_Score failed")

    def score_hamming(self, doc_table, qdata: bytes):
        buf = (C.c_uint8 * max(1, len(qdata))).from_buffer_copy(qdata or b"\0")
        if self.L.II_ScoreHamming(self.h, doc_table.h, buf, len(qdata)) != 0:
            raise RuntimeError("II_ScoreHamming failed")

    def fetch(self, want_freqs=True):
        m = len(self)
        ids = np.zeros(m, dtype=np.uint64)
        scores = np.zeros(m, dtype=np.float64)
        n = self.L.II_ResultSet_NumChildren(self.h)
        freqs = np.zeros((n, m), dtype=np.uint32) if want_freqs else None
        rc = self.L.II_ResultSet_Fetch(self.h, _ptr(ids), _ptr(scores), _ptr(freqs) if want_freqs else None)
        if rc != 0:
            raise RuntimeError("II_ResultSet_Fetch failed")
        return ids, scores, freqs

    def topn(self, n):
        ids = np.zeros(n, dtype=np.uint64)
        scores = np.zeros(n, dtype=np.float64)
        got = self.L.II_ResultSet_TopN(self.h, n, _ptr(ids), _ptr(scores))
        return ids[:got], scores[:got]

    def into_child(self, terms, weight=1.0, with_positions=False):
        """II_ResultSet_IntoChild: this evaluated AND / OR becomes ONE child (a PostingList view) of another aggregate; terms =
        (weight, idf, bm25_idf) of ITS children in their original order.  The result set is consumed."""
        arr = (II_TermParams * len(terms))(*[II_TermParams(*t) for t in terms])
        h = self.L.II_ResultSet_IntoChild(self.h, arr, weight, int(with_positions))
        self.h = None
        if not h:
            raise RuntimeError("II_ResultSet_IntoChild failed")
        return PostingList(h)

    def into_iterator(self, weight=1.0):
        it = self.L.II_NewResultIterator(self.h, weight)
        self.h = None  # ownership moved
        return it

    def close(self):
        if self.h:
            self.L.II_ResultSet_Free(self.h)
            self.h = None

    def free_after(self, stream=None):
        """II_ResultSet_FreeAfter: released once the work enqueued on `stream` (a torch.cuda.Stream, a raw cudaStream_t or None =
        the legacy default stream) so far is done; the host does not wait."""
        if self.h:
            self.L.II_ResultSet_FreeAfter(self.h, _stream_handle(stream))
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _stream_handle(stream):
    if stream is None:
        return None
    return C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)


def intersect_batch_device(batch, stream=None):
    """II_IntersectBatchDevice: batch[i] = the posting lists of query i's AND.  Enqueued without a host wait; `stream` waits for
    every AND.  Returns [(ResultSet or None, device docId pointer, device count pointer, cap)] per query; a None set has cap 0."""
    nq = len(batch)
    arrays = [_list_array(lists) if lists else None for lists in batch]
    lists_pp = (C.c_void_p * max(1, nq))(*[C.cast(a, C.c_void_p) if a is not None else None for a in arrays])
    n_lists = (C.c_size_t * max(1, nq))(*[len(lists) for lists in batch])
    out = (C.c_void_p * max(1, nq))()
    L = lib()
    L.II_IntersectBatchDevice(nq, lists_pp, n_lists, _stream_handle(stream), out)
    res = []
    for i in range(nq):
        if not out[i]:
            res.append((None, None, None, 0))
            continue
        rs = ResultSet(out[i])
        res.append((rs, L.II_ResultSet_DeviceDocIds(rs.h), L.II_ResultSet_DeviceLen(rs.h), L.II_ResultSet_Capacity(rs.h)))
    return res


def _pending_sets(rc, out, nq):
    if rc != 0:
        raise ValueError("the batch was refused (too many lists, a NULL or nested list)")
    L, res = lib(), []
    for i in range(nq):
        if not out[i]:
            res.append((None, None, None, 0))
            continue
        rs = ResultSet(out[i])
        res.append((rs, L.II_ResultSet_DeviceDocIds(rs.h), L.II_ResultSet_DeviceLen(rs.h), L.II_ResultSet_Capacity(rs.h)))
    return res


def _handle_table(batch):
    """(pointer table per query, its keep-alive arrays, counts) of batch[i] = a list of objects with .h"""
    nq = len(batch)
    arrays = [(C.c_void_p * len(items))(*[x.h for x in items]) if items else None for items in batch]
    pp = (C.c_void_p * max(1, nq))(*[C.cast(a, C.c_void_p) if a is not None else None for a in arrays])
    counts = (C.c_size_t * max(1, nq))(*[len(items) for items in batch])
    return pp, arrays, counts


def union_batch_device(batch, quick_exit=False, stream=None):
    """II_UnionBatchDevice: batch[i] = the posting lists of query i's OR.  Enqueued without a host wait; `stream` waits for the
    batch.  Returns [(ResultSet or None, device docId pointer, device count pointer, cap)] per query (a None set has cap 0);
    raises ValueError when the batch is refused."""
    nq = len(batch)
    pp, _keep, counts = _handle_table(batch)
    out = (C.c_void_p * max(1, nq))()
    rc = lib().II_UnionBatchDevice(nq, pp, counts, int(quick_exit), _stream_handle(stream), out, None)
    return _pending_sets(rc, out, nq)


def numeric_filter_batch_device(batch, stream=None):
    """II_NumericFilterBatchDevice: batch[i] = (leaves, lo, hi, lo_inclusive, hi_inclusive), leaves = NumericList objects the
    range-tree walk picked.  Returns as union_batch_device."""
    nq = len(batch)
    pp, _keep, counts = _handle_table([b[0] for b in batch])
    ranges = (II_NumericRange * max(1, nq))(*[II_NumericRange(float(lo), float(hi), int(li), int(hi_)) for _, lo, hi, li, hi_ in batch])
    out = (C.c_void_p * max(1, nq))()
    rc = lib().II_NumericFilterBatchDevice(nq, pp, counts, ranges, _stream_handle(stream), out, None)
    return _pending_sets(rc, out, nq)


def _filter_child_table(batch):
    """(pointer table per query, its keep-alive arrays, counts) of batch[q] = [(child, mode)], child = a PostingList, a ResultSet
    or None; a closed or consumed child raises ValueError"""
    nq = len(batch)
    arrays = []
    for items in batch:
        a = (II_FilterChild * max(1, len(items)))()
        for i, (child, mode) in enumerate(items):
            if child is None:
                a[i] = II_FilterChild(None, None, mode)
                continue
            if not isinstance(child, (PostingList, ResultSet)) or not child.h:
                raise ValueError(f"child {i} is neither None nor a live PostingList / ResultSet")
            a[i] = II_FilterChild(child.h, None, mode) if isinstance(child, PostingList) else II_FilterChild(None, child.h, mode)
        arrays.append(a)
    pp = (C.c_void_p * max(1, nq))(*[C.cast(a, C.c_void_p) for a in arrays])
    counts = (C.c_size_t * max(1, nq))(*[len(items) for items in batch])
    return pp, arrays, counts


def intersect_filter_batch_device(batch, stream=None):
    """II_IntersectFilterBatchDevice: batch[q] = [(child, mode)] of query q's filter-mode AND, child = a PostingList, a ResultSet
    (pending or settled, e.g. from union_batch_device) or None (an empty child), mode 0 = required, 1 = NOT.  The children are
    borrowed.  Returns as union_batch_device; raises ValueError when the batch is refused or a child is closed or consumed (only
    None stands for an empty child)."""
    nq = len(batch)
    pp, _keep, counts = _filter_child_table(batch)
    out = (C.c_void_p * max(1, nq))()
    rc = lib().II_IntersectFilterBatchDevice(nq, pp, counts, _stream_handle(stream), out, None)
    return _pending_sets(rc, out, nq)


def union_filter_batch_device(batch, stream=None):
    """II_UnionFilterBatchDevice: batch[q] = the children of query q's filter-mode OR, each a PostingList, a ResultSet (pending
    or settled, e.g. from intersect_filter_batch_device or numeric_filter_batch_device) or None (an empty child).  The children
    are borrowed.  Returns as union_batch_device; raises ValueError when the batch is refused or a child is closed or consumed
    (only None stands for an empty child)."""
    nq = len(batch)
    pp, _keep, counts = _filter_child_table([[(c, 0) for c in items] for items in batch])
    out = (C.c_void_p * max(1, nq))()
    rc = lib().II_UnionFilterBatchDevice(nq, pp, counts, _stream_handle(stream), out, None)
    return _pending_sets(rc, out, nq)


def intersect(lists) -> ResultSet:
    return ResultSet(lib().II_Intersect(_list_array(lists), len(lists)))


def intersect_ex(lists, modes) -> ResultSet:
    """II_IntersectEx: modes[i] 0 = required, 1 = NOT, 2 = OPTIONAL"""
    return ResultSet(lib().II_IntersectEx(_list_array(lists), (C.c_int * len(lists))(*modes), len(lists)))


def postings_with_offsets(block_lists, codec=0):
    """II_PostingList_FromBlocksBatchOffsets: block_lists[i] = list of (first, last, n, bytes) of term i (Full codec); the term
    positions stay on the device for II_IntersectPhrase"""
    views, keep = [], []
    for blocks in block_lists:
        arr = (II_BlockView * max(1, len(blocks)))()
        for i, (first, last, n, data) in enumerate(blocks):
            buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
            keep.append(buf)
            arr[i] = II_BlockView(first, last, n, C.cast(buf, C.POINTER(C.c_uint8)), len(data))
        views.append(arr)
    n = len(block_lists)
    ptrs = (C.c_void_p * n)(*[C.cast(v, C.c_void_p) for v in views])
    ns = (C.c_size_t * n)(*[len(b) for b in block_lists])
    out = (C.c_void_p * n)()
    if lib().II_PostingList_FromBlocksBatchOffsets(n, ptrs, ns, codec, out) != n:
        raise RuntimeError("batch decode failed")
    return [PostingList(h) for h in out]


def intersect_phrase(lists, max_slop, in_order, modes=None) -> ResultSet:
    """II_IntersectPhrase: max_slop None = no limit"""
    m = (C.c_int * len(lists))(*modes) if modes is not None else None
    return ResultSet(lib().II_IntersectPhrase(_list_array(lists), m, len(lists), -1 if max_slop is None else int(max_slop), int(in_order)))


def union(lists, quick_exit=False) -> ResultSet:
    return ResultSet(lib().II_Union(_list_array(lists), len(lists), int(quick_exit)))


def search_topn(lists, is_union, scorer, terms, agg_weight, num_docs, avg_doc_len, doc_table, top_n):
    arr = (II_TermParams * len(terms))(*[II_TermParams(*t) for t in terms])
    st = II_IndexStats(num_docs, 0, avg_doc_len)
    ids = np.zeros(top_n, dtype=np.uint64)
    scores = np.zeros(top_n, dtype=np.float64)
    total = C.c_size_t(0)
    got = lib().II_SearchTopN(_list_array(lists), len(lists), int(is_union), scorer, arr, agg_weight, C.byref(st),
                              doc_table.h if doc_table else None, top_n, _ptr(ids), _ptr(scores), C.byref(total))
    return ids[:got], scores[:got], total.value


class SearchBatch:
    """Argument block of II_SearchTopNBatch, built once and reusable: queries = [(lists, terms), ...]."""

    def __init__(self, queries, top_n):
        self.nq, self.top_n = len(queries), top_n
        self._keep = []
        self.lists = (C.c_void_p * self.nq)()
        self.terms = (C.c_void_p * self.nq)()
        self.n_lists = (C.c_size_t * self.nq)()
        for i, (lists, terms) in enumerate(queries):
            la = _list_array(lists)
            ta = (II_TermParams * len(terms))(*[II_TermParams(*t) for t in terms])
            self._keep += [la, ta, lists]
            self.lists[i] = C.cast(la, C.c_void_p)
            self.terms[i] = C.cast(ta, C.c_void_p)
            self.n_lists[i] = len(lists)
        self.ids = np.zeros((self.nq, top_n), dtype=np.uint64)
        self.scores = np.zeros((self.nq, top_n), dtype=np.float64)
        self.counts = np.zeros(self.nq, dtype=np.uint64)
        self.totals = np.zeros(self.nq, dtype=np.uint64)

    def run(self, is_union, scorer, agg_weight, num_docs, avg_doc_len, doc_table):
        st = II_IndexStats(num_docs, 0, avg_doc_len)
        rc = lib().II_SearchTopNBatch(self.nq, self.lists, self.n_lists, int(is_union), scorer, self.terms, agg_weight, C.byref(st),
                                      doc_table.h if hasattr(doc_table, "h") else doc_table, self.top_n, _ptr(self.ids),
                                      _ptr(self.scores), _ptr(self.counts), _ptr(self.totals))
        if rc != 0:
            raise RuntimeError("II_SearchTopNBatch failed")
        return [(self.ids[i, :int(self.counts[i])].copy(), self.scores[i, :int(self.counts[i])].copy(), int(self.totals[i]))
                for i in range(self.nq)]


def stats(reset=False) -> II_Stats:
    return lib().II_GetStats(reset)


def smoke(ol) -> None:
    """Tiny 3-term AND + BM25STD on cuda:0, checked against the oracle (called by __graft_entry__.smoke)."""
    rng = np.random.default_rng(5)
    n_docs = 200_000
    lists = [np.unique(rng.integers(1, n_docs, m)).astype(np.uint64) for m in (40_000, 90_000, 15_000)]
    freqs = [rng.integers(1, 9, len(l)).astype(np.uint32) for l in lists]
    doc_len = rng.integers(50, 500, n_docs + 1).astype(np.uint32)
    idx = [ol.InvIndex(ol.CODEC_FREQS_ONLY, l, f) for l, f in zip(lists, freqs)]
    pls = [PostingList.from_blocks(ix.blocks(), CODEC_FREQS_ONLY) for ix in idx]
    rs = intersect(pls)
    exp = ol.run_intersect(idx)
    terms = [(1.0, ol.postings().orc_idf(n_docs, len(l)), ol.postings().orc_idf_bm25(n_docs, len(l))) for l in lists]
    avg = float(doc_len[1:].mean())
    rs.score(SCORER_BM25STD, terms, 1.0, n_docs, avg, DocTable(n_docs, doc_len))
    ids, scores, fr = rs.fetch()
    assert ids.tolist() == [e[0] for e in exp], "docID sequence differs from the oracle"
    order = rs.child_order().tolist()
    for i in range(0, len(exp), max(1, len(exp) // 50)):
        doc, ch = exp[i]
        assert [c for c, _ in ch] == order
        s = ol.oracle_score(ol.SCORER_BM25STD, [f for _, f in ch], [terms[c][1] for c, _ in ch], [terms[c][2] for c, _ in ch],
                            [1.0] * len(ch), 1.0, int(doc_len[doc]), 1, 1.0, n_docs, avg)
        assert np.float64(s).tobytes() == np.float64(scores[i]).tobytes(), (s, scores[i])
    # the fused batch route (II_SearchTopNBatch: window pre-pass + membership + scorer + top-N for every query of the batch):
    # top-10 of the same AND and of two 2-term ANDs, ranked (score desc, docId asc) like RPSorter
    dt = DocTable(n_docs, doc_len)
    combos = [(0, 1, 2), (0, 1), (1, 2)]
    batch = SearchBatch([([pls[c] for c in cb], [terms[c] for c in cb]) for cb in combos], 10)
    out = batch.run(False, SCORER_BM25STD, 1.0, n_docs, avg, dt)
    for cb, (bids, bscores, total) in zip(combos, out):
        r2 = intersect([pls[c] for c in cb])
        r2.score(SCORER_BM25STD, [terms[c] for c in cb], 1.0, n_docs, avg, dt)
        i2, s2, _ = r2.fetch()
        top = np.lexsort((i2, -s2))[:10]
        assert total == len(i2) and bids.tolist() == i2[top].tolist(), "fused batch top-N differs from the per-query chain"
        assert bscores.tobytes() == s2[top].tobytes()
    print(f"smoke postings ok: {len(ids)} hits of 3-term AND, BM25STD bit-equal to the oracle; fused batch top-10 of {len(combos)} queries equal")
