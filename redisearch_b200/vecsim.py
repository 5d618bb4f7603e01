"""ctypes face of libvecsim_b200.so, mirroring the reference's VecSim C API names
(deps/VectorSimilarity/src/VecSim/vec_sim.h, query_results.h) so the parity tests read like the
reference's own tests (tests/unit/test_bruteforce.cpp).  No compute happens here.
"""
import ctypes as C

import numpy as np

from ._lib import load_library

# enum values — include/vecsim_b200.h (== VS/vec_sim_common.h:60-87, query_results.h:21-26)
VecSimType_FLOAT32, VecSimType_FLOAT64, VecSimType_BFLOAT16, VecSimType_FLOAT16 = 0, 1, 2, 3
VecSimType_INT8, VecSimType_UINT8 = 4, 5
VecSimAlgo_BF = 0
VecSimMetric_L2, VecSimMetric_IP, VecSimMetric_Cosine = 0, 1, 2
BY_SCORE, BY_ID, BY_SCORE_THEN_ID = 0, 1, 2
VecSim_QueryReply_OK, VecSim_QueryReply_TimedOut = 0, 1
QUERY_TYPE_NONE, QUERY_TYPE_KNN, QUERY_TYPE_HYBRID, QUERY_TYPE_RANGE = 0, 1, 2, 3
EMPTY_MODE, STANDARD_KNN, HYBRID_ADHOC_BF, HYBRID_BATCHES, HYBRID_BATCHES_TO_ADHOC_BF, RANGE_QUERY = range(6)

ELEM_SIZE = {VecSimType_FLOAT32: 4, VecSimType_BFLOAT16: 2, VecSimType_FLOAT16: 2, VecSimType_INT8: 1,
             VecSimType_UINT8: 1}


class BFParams(C.Structure):
    _fields_ = [("type", C.c_int), ("dim", C.c_size_t), ("metric", C.c_int), ("multi", C.c_bool),
                ("initialCapacity", C.c_size_t), ("blockSize", C.c_size_t)]


class _AlgoParams(C.Union):  # sizeof == 120 (SVSParams is the widest arm), tests/golden/vecsim_abi_layout.txt
    _fields_ = [("bfParams", BFParams), ("_pad", C.c_uint8 * 120)]


class VecSimParams(C.Structure):
    _fields_ = [("algo", C.c_int), ("algoParams", _AlgoParams), ("logCtx", C.c_void_p)]


class VecSimQueryParams(C.Structure):
    _fields_ = [("_runtime", C.c_uint8 * 32), ("batchSize", C.c_size_t), ("searchMode", C.c_int),
                ("timeoutCtx", C.c_void_p)]


class VecSimRawParam(C.Structure):
    _fields_ = [("name", C.c_char_p), ("nameLen", C.c_size_t), ("value", C.c_char_p), ("valLen", C.c_size_t)]


class VecSimIndexBasicInfo(C.Structure):
    _fields_ = [("algo", C.c_int), ("metric", C.c_int), ("type", C.c_int), ("isMulti", C.c_bool),
                ("isTiered", C.c_bool), ("isDisk", C.c_bool), ("blockSize", C.c_size_t), ("dim", C.c_size_t)]


class VecSimIndexStatsInfo(C.Structure):
    _fields_ = [("memory", C.c_size_t), ("numberOfMarkedDeleted", C.c_size_t),
                ("directHNSWInsertions", C.c_size_t), ("flatBufferSize", C.c_size_t)]


class _FieldValue(C.Union):
    _fields_ = [("floatingPointValue", C.c_double), ("integerValue", C.c_int64), ("uintegerValue", C.c_uint64),
                ("stringValue", C.c_char_p), ("iteratorValue", C.c_void_p)]


class CommonInfo(C.Structure):
    _fields_ = [("basicInfo", VecSimIndexBasicInfo), ("indexSize", C.c_size_t), ("indexLabelCount", C.c_size_t), ("memory", C.c_uint64),
                ("lastMode", C.c_int)]


class VecSimIndexDebugInfo(C.Structure):
    """vec_sim_common.h:449-457; the union behind commonInfo is carried as opaque bytes (a FLAT index fills bfInfo only)"""
    _fields_ = [("commonInfo", CommonInfo), ("_union", C.c_uint8 * 296)]


class VecSim_InfoField(C.Structure):
    _fields_ = [("fieldName", C.c_char_p), ("fieldType", C.c_int), ("fieldValue", _FieldValue)]


class VecSimB200_Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("scan_launches", C.c_uint64), ("scan_device_us", C.c_double),
                ("scan_bytes", C.c_uint64)]


TIMEOUT_CB = C.CFUNCTYPE(C.c_int, C.c_void_p)
LOG_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_char_p, C.c_char_p)

# every symbol include/vecsim_b200.h declares: (name, restype, argtypes)
_P, _SZ = C.c_void_p, C.c_size_t
SIGNATURES = [
    ("VecSimIndex_New", _P, [C.POINTER(VecSimParams)]),
    ("VecSimIndex_EstimateInitialSize", _SZ, [C.POINTER(VecSimParams)]),
    ("VecSimIndex_EstimateElementSize", _SZ, [C.POINTER(VecSimParams)]),
    ("VecSimIndex_Free", None, [_P]),
    ("VecSimIndex_AddVector", C.c_int, [_P, _P, _SZ]),
    ("VecSimIndex_DeleteVector", C.c_int, [_P, _SZ]),
    ("VecSimIndex_IndexSize", _SZ, [_P]),
    ("VecSimIndex_TopKQuery", _P, [_P, _P, _SZ, C.POINTER(VecSimQueryParams), C.c_int]),
    ("VecSimIndex_RangeQuery", _P, [_P, _P, C.c_double, C.POINTER(VecSimQueryParams), C.c_int]),
    ("VecSimIndex_GetDistanceFrom_Unsafe", C.c_double, [_P, _SZ, _P]),
    ("VecSimIndex_PreferAdHocSearch", C.c_bool, [_P, _SZ, _SZ, C.c_bool]),
    ("VecSimIndex_ResolveParams", C.c_int, [_P, C.POINTER(VecSimRawParam), C.c_int, C.POINTER(VecSimQueryParams), C.c_int]),
    ("VecSimBatchIterator_New", _P, [_P, _P, C.POINTER(VecSimQueryParams)]),
    ("VecSimBatchIterator_Next", _P, [_P, _SZ, C.c_int]),
    ("VecSimBatchIterator_HasNext", C.c_bool, [_P]),
    ("VecSimBatchIterator_Reset", None, [_P]),
    ("VecSimBatchIterator_Free", None, [_P]),
    ("VecSimIndex_AdhocBfCtx_New", _P, [_P, _P]),
    ("VecSimIndex_AdhocBfCtx_Free", None, [_P]),
    ("VecSimIndex_AdhocBfCtx_GetDistanceFrom", C.c_double, [_P, _SZ]),
    ("VecSimIndex_AdhocBfCtx_GetExactDistances", None, [_P, _P, _P, _SZ]),
    ("VecSimQueryReply_Len", _SZ, [_P]),
    ("VecSimQueryReply_GetCode", C.c_int, [_P]),
    ("VecSimQueryReply_Free", None, [_P]),
    ("VecSimQueryReply_GetIterator", _P, [_P]),
    ("VecSimQueryReply_IteratorNext", _P, [_P]),
    ("VecSimQueryReply_IteratorHasNext", C.c_bool, [_P]),
    ("VecSimQueryReply_IteratorReset", None, [_P]),
    ("VecSimQueryReply_IteratorFree", None, [_P]),
    ("VecSimQueryResult_GetId", C.c_int64, [_P]),
    ("VecSimQueryResult_GetScore", C.c_double, [_P]),
    ("VecSim_Normalize", None, [_P, _SZ, C.c_int]),
    ("VecSimParams_GetQueryBlobSize", _SZ, [C.c_int, _SZ, C.c_int]),
    ("VecSimIndex_BasicInfo", VecSimIndexBasicInfo, [_P]),
    ("VecSimIndex_StatsInfo", VecSimIndexStatsInfo, [_P]),
    ("VecSimIndex_DebugInfo", VecSimIndexDebugInfo, [_P]),
    ("VecSimB200_TopKFilteredBatch", C.c_int, [_P, _P, _SZ, _SZ, _P, _P, _P, _P, _P]),
    ("VecSimB200_TopKFilteredBatchDevice", C.c_int, [_P, _P, _SZ, _SZ, _P, _P, _P, _P, _P, _P, _P]),
    ("VecSimB200_HybridTopKBatchDevice", C.c_int, [_P, _P, _SZ, _SZ, _P, _P, _P, C.POINTER(VecSimQueryParams), _P, _P, _P, _P, _P]),
    ("VecSimIndex_DebugInfoIterator", _P, [_P]),
    ("VecSimDebugInfoIterator_NumberOfFields", _SZ, [_P]),
    ("VecSimDebugInfoIterator_HasNextField", C.c_bool, [_P]),
    ("VecSimDebugInfoIterator_NextField", C.POINTER(VecSim_InfoField), [_P]),
    ("VecSimDebugInfoIterator_Free", None, [_P]),
    ("VecSimTieredIndex_GC", None, [_P]),
    ("VecSimTieredIndex_AcquireSharedLocks", None, [_P]),
    ("VecSimTieredIndex_ReleaseSharedLocks", None, [_P]),
    ("VecSim_SetTimeoutCallbackFunction", None, [TIMEOUT_CB]),
    ("VecSim_SetLogCallbackFunction", None, [LOG_CB]),
    ("VecSim_SetWriteMode", None, [C.c_int]),
    ("VecSim_SetTestLogContext", None, [C.c_char_p, C.c_char_p]),
    ("VecSim_UpdateThreadPoolSize", None, [_SZ]),
    ("VecSim_GetSharedMemory", _SZ, []),
    ("VecSimB200_TopKQueryBatch", C.c_int, [_P, _P, _SZ, _SZ, _SZ, C.POINTER(VecSimQueryParams), _P, _P]),
    ("VecSimB200_TopKQueryBatchDevice", C.c_int, [_P, _P, _SZ, _SZ, _P, _P, _P]),
    ("VecSimB200_RangeQueryBatchDevice", C.c_int, [_P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, _P, _P]),
    ("VecSimB200_LabelRangeQueryBatchDevice", C.c_int, [_P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, _P, _P]),
    ("VecSimB200_HybridRangeQueryBatchDevice", C.c_int,
     [_P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, _P, C.POINTER(VecSimQueryParams), _P, _P, _P, _P, _P]),
    ("VecSimB200_RangeQueryBatch", C.c_int, [_P, _P, _SZ, _SZ, _P, C.POINTER(VecSimQueryParams), C.c_int, _P, _P]),
    ("VecSimB200_AddVectors", C.c_int, [_P, _P, _SZ, _SZ, _P, _SZ]),
    ("VecSimB200_AddVectorsDevice", C.c_int, [_P, _P, _SZ, _SZ]),
    ("VecSimB200_Reserve", C.c_int, [_P, _SZ]),
    ("VecSimB200_Flush", C.c_int, [_P]),
    ("VecSimB200_DeviceRows", _P, [_P, C.POINTER(_SZ), C.POINTER(_SZ)]),
    ("VecSimB200_GetStats", VecSimB200_Stats, [_P, C.c_bool]),
    ("VecSimB200_ReadRows", C.c_int, [_P, _SZ, _SZ, _P]),
    ("VecSimB200_MergeShardTopK", C.c_int, [_P, _P, _SZ, _SZ, _SZ, _P, _P, _P]),
    ("VecSimB200_TopKFiltered", C.c_int, [_P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, C.POINTER(_SZ)]),
    ("VecSimB200_HybridTopK", C.c_int, [_P, _P, _SZ, _P, C.POINTER(VecSimQueryParams), _P, _P, C.POINTER(_SZ), C.POINTER(C.c_int), C.POINTER(_SZ)]),
    ("VecSimB200_LastBatchPath", C.c_int, [_P]),
    ("VecSimB200_LastCoarseShadowBits", C.c_int, [_P]),
    ("VecSimB200_SetCoarseMode", None, [C.c_int]),
    ("VecSimB200_LastCoarseFlags", C.c_int, [_P, _P, _SZ]),
    ("VecSimB200_Version", C.c_char_p, []),
    ("VecSimB200_ShardBlockBytes", _SZ, [_SZ, _SZ]),
    ("VecSimB200_MergeShardBlocks", C.c_int, [_P, _SZ, _SZ, _SZ, _P, _P, _P]),
    ("VecSimB200_ShardGroup_UniqueId", C.c_int, [_P]),
    ("VecSimB200_ShardGroup_New", _P, [_P, C.c_int, C.c_int]),
    ("VecSimB200_ShardGroup_Free", None, [_P]),
    ("VecSimB200_ShardGroup_Rank", C.c_int, [_P]),
    ("VecSimB200_ShardGroup_Size", C.c_int, [_P]),
    ("VecSimB200_ShardGroup_TopKBatchDevice", C.c_int, [_P, _P, _P, _SZ, _SZ, _P, _P, _P]),
    ("VecSimB200_ShardGroup_TopKBatch", C.c_int, [_P, _P, _P, _SZ, _SZ, _SZ, _P, _P]),
    ("VecSimB200_ShardListBlockBytes", _SZ, [_SZ, _SZ]),
    ("VecSimB200_MergeShardListBlocks", C.c_int, [_P, _SZ, _SZ, _SZ, C.c_int, C.c_int, _P, _P, _P, _P]),
    ("VecSimB200_ShardGroup_HybridTopKBatchDevice", C.c_int,
     [_P, _P, _P, _SZ, _SZ, _P, _P, _P, C.POINTER(VecSimQueryParams), _P, _P, _P, _P, _P]),
    ("VecSimB200_ShardGroup_RangeQueryBatchDevice", C.c_int, [_P, _P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, _P, _P]),
    ("VecSimB200_ShardGroup_HybridRangeQueryBatchDevice", C.c_int,
     [_P, _P, _P, _SZ, _P, _SZ, C.c_int, _P, _P, _P, C.POINTER(VecSimQueryParams), _P, _P, _P, _P, _P]),
]
# VecSim_SetMemoryFunctions takes a struct by value; declared in the header, bound lazily.
EXTRA_SYMBOLS = ["VecSim_SetMemoryFunctions"]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = load_library("libvecsim_b200.so")
        for name, res, args in SIGNATURES:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class VecSimIndex:
    """A FLAT index living in HBM.  Methods are the C API calls with numpy in/out."""

    def __init__(self, vtype, dim, metric, multi=False, block_size=1024, initial_capacity=0):
        self.L = lib()
        p = VecSimParams()
        p.algo = VecSimAlgo_BF
        p.algoParams.bfParams = BFParams(vtype, dim, metric, multi, initial_capacity, block_size)
        self.vtype, self.dim, self.metric, self.multi = vtype, dim, metric, multi
        self.h = self.L.VecSimIndex_New(C.byref(p))
        if not self.h:
            raise RuntimeError("VecSimIndex_New returned NULL (no CUDA device, or unsupported parameters)")

    def close(self):
        if self.h:
            self.L.VecSimIndex_Free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- mutation
    def add(self, blob: np.ndarray, label: int) -> int:
        blob = np.ascontiguousarray(blob)
        return self.L.VecSimIndex_AddVector(self.h, _ptr(blob), label)

    def add_many(self, blobs: np.ndarray, labels=None, label0=0) -> int:
        blobs = np.ascontiguousarray(blobs)
        lab = None
        if labels is not None:
            lab = np.ascontiguousarray(labels, dtype=np.uint64)
        return self.L.VecSimB200_AddVectors(self.h, _ptr(blobs), blobs.strides[0], blobs.shape[0],
                                            _ptr(lab) if lab is not None else None, label0)

    def delete(self, label: int) -> int:
        return self.L.VecSimIndex_DeleteVector(self.h, label)

    def size(self) -> int:
        return self.L.VecSimIndex_IndexSize(self.h)

    # -- queries
    def _drain(self, rep):
        n = self.L.VecSimQueryReply_Len(rep)
        code = self.L.VecSimQueryReply_GetCode(rep)
        ids = np.empty(n, dtype=np.int64)
        scores = np.empty(n, dtype=np.float64)
        it = self.L.VecSimQueryReply_GetIterator(rep)
        i = 0
        while self.L.VecSimQueryReply_IteratorHasNext(it):
            item = self.L.VecSimQueryReply_IteratorNext(it)
            ids[i] = self.L.VecSimQueryResult_GetId(item)
            scores[i] = self.L.VecSimQueryResult_GetScore(item)
            i += 1
        assert i == n
        self.L.VecSimQueryReply_IteratorFree(it)
        self.L.VecSimQueryReply_Free(rep)
        return ids, scores, code

    def topk(self, q: np.ndarray, k: int, order=BY_SCORE, params=None):
        q = np.ascontiguousarray(q)
        rep = self.L.VecSimIndex_TopKQuery(self.h, _ptr(q), k, params, order)
        return self._drain(rep)

    def range(self, q: np.ndarray, radius: float, order=BY_SCORE, params=None):
        q = np.ascontiguousarray(q)
        rep = self.L.VecSimIndex_RangeQuery(self.h, _ptr(q), radius, params, order)
        if not rep:
            raise ValueError("VecSimIndex_RangeQuery rejected its arguments")
        return self._drain(rep)

    def topk_batch(self, qs: np.ndarray, k: int, params=None):
        qs = np.ascontiguousarray(qs)
        nq = qs.shape[0]
        labels = np.empty((nq, k), dtype=np.uint64)
        scores = np.empty((nq, k), dtype=np.float64)
        rc = self.L.VecSimB200_TopKQueryBatch(self.h, _ptr(qs), qs.strides[0], nq, k, params, _ptr(labels), _ptr(scores))
        return labels, scores, rc

    def range_batch(self, qs: np.ndarray, radii, order=BY_SCORE, params=None):
        """nq range queries in one call: ([(ids, scores, code) per query], rc, flags); flags[i] = 1 if query i was answered
        by the tensor-core route.  rc == -1 (invalid order, negative radius, device failure): no replies, an empty list."""
        qs = np.ascontiguousarray(qs)
        nq = qs.shape[0]
        radii = np.ascontiguousarray(np.broadcast_to(np.asarray(radii, dtype=np.float64), (nq,)))
        reps = (C.c_void_p * max(1, nq))()
        flags = np.zeros(nq, dtype=np.uint32)
        rc = self.L.VecSimB200_RangeQueryBatch(self.h, _ptr(qs), qs.strides[0], nq, _ptr(radii), params, order, C.cast(reps, C.c_void_p),
                                               _ptr(flags))
        if rc == -1:
            return [], rc, flags
        return [self._drain(reps[i]) for i in range(nq)], rc, flags

    def topk_filtered(self, q: np.ndarray, k: int, doc_ids, n=None):
        """k nearest among the listed labels.  doc_ids: ascending uint32 numpy array, or a device pointer (int) with n."""
        q = np.ascontiguousarray(q)
        labels = np.zeros(k, dtype=np.uint64)
        scores = np.zeros(k, dtype=np.float64)
        cnt = C.c_size_t(0)
        if isinstance(doc_ids, np.ndarray):
            ids = np.ascontiguousarray(doc_ids, dtype=np.uint32)
            rc = self.L.VecSimB200_TopKFiltered(self.h, _ptr(q), k, _ptr(ids), len(ids), 0, _ptr(labels), _ptr(scores), C.byref(cnt))
        else:
            rc = self.L.VecSimB200_TopKFiltered(self.h, _ptr(q), k, C.c_void_p(int(doc_ids)), n, 1, _ptr(labels), _ptr(scores), C.byref(cnt))
        return labels[:cnt.value], scores[:cnt.value], rc

    def topk_filtered_batch_device(self, d_queries, k, doc_ids, caps, counts=None, out_labels=None, out_scores=None, out_counts=None,
                                   stream=None):
        """VecSimB200_TopKFilteredBatchDevice, enqueued on `stream` (a torch.cuda.Stream, a raw cudaStream_t or None = the legacy
        default stream) without waiting.  d_queries: a [nq, query_pitch] CUDA tensor of stored-form blobs (or a device pointer);
        doc_ids / counts: per query a device pointer (int) or None; caps: per query the host bound.  Outputs are torch CUDA tensors
        ([nq, k] int64 / float32, [nq] int32 holding the u32 counts), allocated when not given.  Returns (labels, scores, counts, rc)."""
        import torch

        nq = len(caps)
        dev = torch.device("cuda")
        if out_labels is None:
            out_labels = torch.empty((nq, k), dtype=torch.int64, device=dev)
        if out_scores is None:
            out_scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
        if out_counts is None:
            out_counts = torch.empty(nq, dtype=torch.int32, device=dev)
        n = max(1, nq)
        ids = (C.c_void_p * n)(*[int(p) if p else None for p in doc_ids])
        cnt = (C.c_void_p * n)(*[int(p) if p else None for p in counts]) if counts is not None else None
        cap_arr = (C.c_size_t * n)(*[int(c) for c in caps])
        qp = d_queries.data_ptr() if hasattr(d_queries, "data_ptr") else int(d_queries)
        sh = None if stream is None else C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)
        rc = self.L.VecSimB200_TopKFilteredBatchDevice(self.h, C.c_void_p(qp), nq, k, ids, cnt, cap_arr, C.c_void_p(out_labels.data_ptr()),
                                                       C.c_void_p(out_scores.data_ptr()), C.c_void_p(out_counts.data_ptr()), sh)
        return out_labels, out_scores, out_counts, rc

    def hybrid_topk_batch_device(self, d_queries, k, doc_ids, caps, counts=None, params=None, out_labels=None, out_scores=None,
                                 out_counts=None, stream=None):
        """VecSimB200_HybridTopKBatchDevice: topk_filtered_batch_device's arguments and rows, each query on the ragged gather or
        the filtered tensor-core route.  params: a VecSimQueryParams whose searchMode picks the policy (None = automatic).
        Returns (labels, scores, counts, modes, rc); modes[i] = HYBRID_ADHOC_BF or HYBRID_BATCHES, the route query i took."""
        import torch

        nq = len(caps)
        dev = torch.device("cuda")
        if out_labels is None:
            out_labels = torch.empty((nq, k), dtype=torch.int64, device=dev)
        if out_scores is None:
            out_scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
        if out_counts is None:
            out_counts = torch.empty(nq, dtype=torch.int32, device=dev)
        n = max(1, nq)
        ids = (C.c_void_p * n)(*[int(p) if p else None for p in doc_ids])
        cnt = (C.c_void_p * n)(*[int(p) if p else None for p in counts]) if counts is not None else None
        cap_arr = (C.c_size_t * n)(*[int(c) for c in caps])
        modes = np.zeros(n, dtype=np.int32)
        qp = d_queries.data_ptr() if hasattr(d_queries, "data_ptr") else int(d_queries)
        sh = None if stream is None else C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)
        rc = self.L.VecSimB200_HybridTopKBatchDevice(self.h, C.c_void_p(qp), nq, k, ids, cnt, cap_arr,
                                                     C.byref(params) if params is not None else None, C.c_void_p(out_labels.data_ptr()),
                                                     C.c_void_p(out_scores.data_ptr()), C.c_void_p(out_counts.data_ptr()), _ptr(modes), sh)
        return out_labels, out_scores, out_counts, modes[:nq], rc

    def range_batch_device(self, d_queries, d_radii, cap, order=BY_SCORE, out_labels=None, out_scores=None, out_counts=None, stream=None):
        """VecSimB200_RangeQueryBatchDevice, enqueued on `stream` (a torch.cuda.Stream, a raw cudaStream_t or None = the legacy
        default stream) without waiting.  d_queries: a [nq, query_pitch] CUDA tensor of stored-form blobs; d_radii: a [nq] float32
        CUDA tensor.  Outputs are torch CUDA tensors ([nq, cap] int64 / float32, [nq] int32 holding the u32 counts), allocated when
        not given.  Returns (labels, scores, counts, rc)."""
        return self._range_device(self.L.VecSimB200_RangeQueryBatchDevice, d_queries, d_radii, cap, order, out_labels, out_scores,
                                  out_counts, stream)

    def label_range_batch_device(self, d_queries, d_radii, cap, order=BY_SCORE, out_labels=None, out_scores=None, out_counts=None,
                                 stream=None):
        """VecSimB200_LabelRangeQueryBatchDevice: range_batch_device answered per label, on multi-value indexes too (one entry per
        label at its best passing row, counts in labels).  Returns (labels, scores, counts, rc); rc -2 = labels too sparse."""
        return self._range_device(self.L.VecSimB200_LabelRangeQueryBatchDevice, d_queries, d_radii, cap, order, out_labels, out_scores,
                                  out_counts, stream)

    def hybrid_range_batch_device(self, d_queries, d_radii, cap, doc_ids, caps, counts=None, order=BY_SCORE, params=None, out_labels=None,
                                  out_scores=None, out_counts=None, stream=None):
        """VecSimB200_HybridRangeQueryBatchDevice: label_range_batch_device restricted to a filter per query.  doc_ids / counts / caps
        as in hybrid_topk_batch_device; params: a VecSimQueryParams whose searchMode picks the policy (None = automatic).  Returns
        (labels, scores, counts, modes, rc); modes[i] = HYBRID_ADHOC_BF or HYBRID_BATCHES, the route query i took."""
        import torch

        nq = len(caps)
        dev = torch.device("cuda")
        if out_labels is None:
            out_labels = torch.empty((nq, max(cap, 0)), dtype=torch.int64, device=dev)
        if out_scores is None:
            out_scores = torch.empty((nq, max(cap, 0)), dtype=torch.float32, device=dev)
        if out_counts is None:
            out_counts = torch.empty(nq, dtype=torch.int32, device=dev)
        n = max(1, nq)
        ids = (C.c_void_p * n)(*[int(p) if p else None for p in doc_ids])
        cnt = (C.c_void_p * n)(*[int(p) if p else None for p in counts]) if counts is not None else None
        cap_arr = (C.c_size_t * n)(*[int(c) for c in caps])
        modes = np.zeros(n, dtype=np.int32)
        qp = d_queries.data_ptr() if hasattr(d_queries, "data_ptr") else int(d_queries)
        rp = d_radii.data_ptr() if hasattr(d_radii, "data_ptr") else int(d_radii)
        sh = None if stream is None else C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)
        rc = self.L.VecSimB200_HybridRangeQueryBatchDevice(self.h, C.c_void_p(qp), nq, C.c_void_p(rp), cap, order, ids, cnt, cap_arr,
                                                           C.byref(params) if params is not None else None, C.c_void_p(out_labels.data_ptr()),
                                                           C.c_void_p(out_scores.data_ptr()), C.c_void_p(out_counts.data_ptr()), _ptr(modes), sh)
        return out_labels, out_scores, out_counts, modes[:nq], rc

    def _range_device(self, fn, d_queries, d_radii, cap, order, out_labels, out_scores, out_counts, stream):
        import torch

        nq = int(d_queries.shape[0])
        dev = torch.device("cuda")
        if out_labels is None:
            out_labels = torch.empty((nq, max(cap, 0)), dtype=torch.int64, device=dev)
        if out_scores is None:
            out_scores = torch.empty((nq, max(cap, 0)), dtype=torch.float32, device=dev)
        if out_counts is None:
            out_counts = torch.empty(nq, dtype=torch.int32, device=dev)
        sh = None if stream is None else C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)
        rc = fn(self.h, C.c_void_p(d_queries.data_ptr()), nq, C.c_void_p(d_radii.data_ptr()), cap, order, C.c_void_p(out_labels.data_ptr()),
                C.c_void_p(out_scores.data_ptr()), C.c_void_p(out_counts.data_ptr()), sh)
        return out_labels, out_scores, out_counts, rc

    def query_pitch(self) -> int:
        """bytes between the stored-form query blobs of a device batch"""
        return (self.L.VecSimParams_GetQueryBlobSize(self.vtype, self.dim, self.metric) + 15) // 16 * 16

    def distance_from(self, label: int, blob: np.ndarray) -> float:
        blob = np.ascontiguousarray(blob)
        return self.L.VecSimIndex_GetDistanceFrom_Unsafe(self.h, label, _ptr(blob))

    def prefer_adhoc(self, subset: int, k: int, initial: bool) -> bool:
        return bool(self.L.VecSimIndex_PreferAdHocSearch(self.h, subset, k, initial))

    def batch_iterator(self, q: np.ndarray, params=None):
        return BatchIterator(self, np.ascontiguousarray(q), params)

    def adhoc_distances(self, q: np.ndarray, labels) -> np.ndarray:
        q = np.ascontiguousarray(q)
        labels = np.ascontiguousarray(labels, dtype=np.uint64)
        out = np.empty(labels.shape[0], dtype=np.float64)
        ctx = self.L.VecSimIndex_AdhocBfCtx_New(self.h, _ptr(q))
        if not ctx:
            raise RuntimeError("VecSimIndex_AdhocBfCtx_New failed")
        self.L.VecSimIndex_AdhocBfCtx_GetExactDistances(ctx, _ptr(labels), _ptr(out), labels.shape[0])
        self.L.VecSimIndex_AdhocBfCtx_Free(ctx)
        return out

    # -- info
    def basic_info(self) -> VecSimIndexBasicInfo:
        return self.L.VecSimIndex_BasicInfo(self.h)

    def stats_info(self) -> VecSimIndexStatsInfo:
        return self.L.VecSimIndex_StatsInfo(self.h)

    def debug_info(self) -> dict:
        it = self.L.VecSimIndex_DebugInfoIterator(self.h)
        out = {}
        while self.L.VecSimDebugInfoIterator_HasNextField(it):
            f = self.L.VecSimDebugInfoIterator_NextField(it).contents
            if f.fieldType == 0:
                out[f.fieldName.decode()] = f.fieldValue.stringValue.decode()
            elif f.fieldType == 3:
                out[f.fieldName.decode()] = f.fieldValue.floatingPointValue
            else:
                out[f.fieldName.decode()] = f.fieldValue.uintegerValue
        self.L.VecSimDebugInfoIterator_Free(it)
        return out

    def stats(self, reset=False) -> VecSimB200_Stats:
        return self.L.VecSimB200_GetStats(self.h, reset)

    def device_rows(self):
        pitch, rows = C.c_size_t(), C.c_size_t()
        p = self.L.VecSimB200_DeviceRows(self.h, C.byref(pitch), C.byref(rows))
        return p, pitch.value, rows.value


class BatchIterator:
    def __init__(self, index: VecSimIndex, q: np.ndarray, params=None):
        self.index = index
        self.L = index.L
        self.h = self.L.VecSimBatchIterator_New(index.h, _ptr(q), params)

    def next(self, n: int, order=BY_SCORE):
        rep = self.L.VecSimBatchIterator_Next(self.h, n, order)
        return self.index._drain(rep)

    def has_next(self) -> bool:
        return bool(self.L.VecSimBatchIterator_HasNext(self.h))

    def reset(self):
        self.L.VecSimBatchIterator_Reset(self.h)

    def free(self):
        if self.h:
            self.L.VecSimBatchIterator_Free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def normalize(blob: np.ndarray, dim: int, vtype: int) -> None:
    """VecSim_Normalize in place (blob must have room for the int8/uint8 norm)."""
    lib().VecSim_Normalize(_ptr(blob), dim, vtype)
