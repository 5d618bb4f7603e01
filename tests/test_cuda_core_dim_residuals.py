"""Every CUDA-core KNN path against the reference, bit for bit, over the dimension residuals of the distance tiles.

DistTile<DT_F32, MT, RT, QT>::run (redisearch_b200/csrc/distance_core.cuh) copies the summation order of the reference's
AVX-512 kernel, and which of its branches run depends on dim: the scalar baseline below 8, a masked multiply of the dim % 16
head, an odd 16-element step when dim % 32 >= 16, then the 32-wide chunks unrolled U at a time (U set by the tile size
V = RT * QT) and a remainder loop.  DistTile8 (int8 / uint8) and DistTile16 (fp16 / bf16) read 16-byte vectors and a
per-lane tail.  Each kernel instantiates the tile with its own shape and finds its query its own way (shared memory, or
read through L1 when a batch's queries do not fit), so each is swept here over one dim list that reaches every class.

  * CPU: the dim list is checked against the constants of distance_core.cuh and plan_scan_topk, restated below; the
    plain int64 reference of the 8-bit distances equals the C restatement of the reference (orc_distance) bit for bit, and
    the fp32 restatement equals the reference's compiled code where that is built and the host has AVX-512F.
  * GPU, fp32 / int8 / uint8: ids and score bits equal to the (score, label) selection over the reference's scores of the
    stored rows, on the single query (fused and unfused), the batch iterator, range, GetDistanceFrom, the ad-hoc context,
    TopKFiltered, exact-scan batches (partial query tiles, partial CTAs, queries through L1), the range batch and the ragged
    device batch; multi-value indexes of all five types on the label-aware scan, gather_min, the ragged batch and
    GetDistanceFrom; and the fp32 tensor-core route's exact rescoring.
  * GPU, fp16 / bf16: bit-equal to the single-value per-row scores and within the derived bound of the fp64 distance
    (test_half_precision_bounds.py) on the paths its own sweep does not reach.
"""
import numpy as np
import pytest

import oracle_lib as ol
from oracle_lib import BF16, COS, F16, F32, I8, IP, L2, U8
from test_half_precision_bounds import (SIZE_MAX, assert_same_bits, bound_cuda_core, check_answer, decode16, device_batch,
                                        exact_distances, flags_of, per_label, reference_fold, selection, single_scan_scores,
                                        stored_query, stored_rows)
from test_hybrid_device_batch import stored_queries
from test_hybrid_device_batch import device_batch as ragged_batch
from test_vecsim_parity import DIM_SWEEP

VT = {F32: 0, BF16: 2, F16: 3, I8: 4, U8: 5}
MT = {L2: 0, IP: 1, COS: 2}
TNAME = {F32: "fp32", F16: "fp16", BF16: "bf16", I8: "int8", U8: "uint8"}
MNAME = {L2: "L2", IP: "IP", COS: "COS"}

# ------------------------------------------------------------------------------------------------------------------
# the constants of the kernels, restated
# ------------------------------------------------------------------------------------------------------------------
LANES = 32
F32_SCALAR_BELOW = 8  # distance_core.cuh DistTile<DT_F32>::run: `if (dim < 8)` -> the scalar baseline on lane 0
F32_CHUNK, F32_HALF = 32, 16  # `res = dim & 31u, r16 = res & 15u`; `if (res >= 16 && lane >= 16)`: the odd 16-step
I8_VEC = 16  # DistTile8::run: `nvec = dim >> 4; // 16 bytes per lane per step`
H16_VEC = 8  # DistTile16::run: `nvec = dim >> 3; // 8 elements = 16 bytes per lane per step`
K_SCAN_WARPS = 8  # vecsim_kernels.cu: `kScanThreads = 256`, `kScanWarps = kScanThreads / 32`
K_MAX_QUERY_SMEM = 96 * 1024  # vecsim_kernels.cu: `kMaxQuerySmem = 96 * 1024`
K_MAX_SCAN_SMEM = 227 * 1024  # vecsim_kernels.cu: `kMaxScanSmem = 227 * 1024`
K_MAX_FUSED = 128  # topk_common.cuh: `kMaxFusedK = 128`


def unroll(v):
    """distance_core.cuh DistTile<DT_F32>::run: `constexpr int U = (V <= 8) ? 8 : (V <= 16 ? 4 : 2);`"""
    return 8 if v <= 8 else (4 if v <= 16 else 2)


# the tile size V = RT * QT of each CUDA-core kernel (vecsim_kernels.cu `using Tile = DistTile<...>`, coarse_tc.cu refine)
KERNEL_V = {"scan_topk 4x1": 4, "scan_topk 4x8": 32, "scan_scores 4x1": 4, "scan_scores_wide 4x8": 32, "gather": 1,
            "gather_ragged": 1, "scan_topk 4x1 labels": 4, "scan_topk 4x8 labels": 32, "gather_min": 1, "gather_ragged multi": 1,
            "refine / range_refine": 1}


def f32_class(dim, v):
    """(residual class, nchunks class) of DistTile<DT_F32> at tile size v; ("scalar", None) below 8."""
    if dim < F32_SCALAR_BELOW:
        return "dim<8", None
    res = dim % F32_CHUNK
    rc = "r0" if res == 0 else "r1-15" if res < F32_HALF else "r16" if res == F32_HALF else "r17-31"
    nchunks, u = (dim - res) // F32_CHUNK, unroll(v)
    nc = "n0" if nchunks == 0 else "n<U" if nchunks < u else "n%U=0" if nchunks % u == 0 else "n>U,n%U!=0"
    return rc, nc


def vec_class(dim, width):
    """(nvec class, tail) of DistTile8 (width 16) / DistTile16 (width 8): nvec < 32, = 32, > 32 and not a multiple of 32."""
    nvec = dim // width
    c = "nvec<32" if nvec < LANES else "nvec=32" if nvec == LANES else "nvec>32,%32!=0" if nvec % LANES else "nvec>32,%32=0"
    return c, "tail" if dim % width else "no tail"


def query_blob_bytes(vtype, metric, dim):
    """vecsim_kernels.cu query_blob_bytes"""
    if vtype == F32:
        return dim * 4
    if vtype in (F16, BF16):
        return dim * 2
    return dim + (4 if metric == COS else 0)


def queries_through_l1(vtype, metric, dim, nq, k, labels=False):
    """vecsim_kernels.cu plan_scan_topk + launch_scan_dml, restated: the batched scan (QT = 8) reads its queries through L1
    when wq * 8 * round16(blob) exceeds kMaxQuerySmem or, with the lists, the shared memory of a CTA.  Label-aware lists
    (multi-value index) hold 16 bytes per slot.  The library exposes no signal of which instantiation ran, so which batches
    take the L1 branch is inferred from this rule, not observed."""
    if nq == 1:
        return False
    qt = 8
    groups = (nq + qt - 1) // qt
    wq = 8 if groups >= 8 else 4 if groups >= 4 else 2 if groups >= 2 else 1
    qs = wq * qt * ((query_blob_bytes(vtype, metric, dim) + 15) // 16 * 16)
    lists = K_SCAN_WARPS * qt * k * (16 if labels else 8) + K_SCAN_WARPS * qt * 12
    return qs > K_MAX_QUERY_SMEM or qs + lists > K_MAX_SCAN_SMEM


# the dims that fill DIM_SWEEP's holes: V = 32 with an even / odd nchunks at residual 16 and 17-31 (80, 95, 112); V <= 8 with
# nchunks = 8 at residual 16 and 17-31 (272, 287) and nchunks = 9 in every residual class (288, 300, 304, 311); int8 nvec = 32
# (512, 513) and nvec > 32 without a tail (800, 1552); and the queries of an int8 / uint8 batch through L1 (1552, 1553)
EXTRA_DIMS = [80, 95, 112, 272, 287, 288, 300, 304, 311, 512, 513, 800, 1552, 1553]
DIMS = sorted(set(DIM_SWEEP) | set(EXTRA_DIMS))
BATCH_NQ = (2, 9, 64, 71)
BATCH_K = (1, 10, 128, 129, 1000)
HALF_DIMS = (3, 17, 100, 257, 300, 304, 771, 1553)  # fp16 / bf16: the ragged batch, 64-query batches, multi-value indexes
MULTI_NQ = (9, 64)
REFINE_DIMS = (40, 56, 72, 288, 304, 1000)  # the fp32 route: dim % 8 == 0, dim >= 32
# which dims reach each kernel in the GPU tests below (fp32); the kernels of the first group are held to every class
SWEPT = {"scan_topk 4x1": DIMS, "scan_topk 4x8": DIMS, "scan_scores 4x1": DIMS, "scan_scores_wide 4x8": DIMS, "gather": DIMS,
         "gather_ragged": DIMS, "scan_topk 4x1 labels": DIMS, "scan_topk 4x8 labels": DIMS, "gather_min": DIMS,
         "gather_ragged multi": DIMS}
PARTIAL = {"refine / range_refine": REFINE_DIMS}


def coverage():
    """{class: first dim (or (dim, nq)) of the GPU tests in it} for every class the kernels distinguish."""
    out = {}
    for kernel, dims in list(SWEPT.items()) + list(PARTIAL.items()):
        v = KERNEL_V[kernel]
        for d in dims:
            out.setdefault(("fp32", kernel, v) + f32_class(d, v), d)
    for d in DIMS:
        out.setdefault(("int8/uint8",) + vec_class(d, I8_VEC), d)
    for d in sorted(set(DIM_SWEEP) | set(HALF_DIMS)):  # DIM_SWEEP: test_half_precision_bounds.py's sweep of the other paths
        out.setdefault(("fp16/bf16",) + vec_class(d, H16_VEC), d)
    for vtype in (F32, F16, BF16, I8, U8):
        for metric in (L2, IP, COS):
            row_dims = HALF_DIMS if vtype in (F16, BF16) else DIMS
            row_nq = (64,) if vtype in (F16, BF16) else BATCH_NQ
            for labels, nqs in ((False, row_nq), (True, MULTI_NQ)):
                for d in row_dims:
                    for nq in nqs:
                        l1 = queries_through_l1(vtype, metric, d, nq, K_MAX_FUSED, labels)
                        out.setdefault((TNAME[vtype], MNAME[metric], "labels" if labels else "rows", "L1" if l1 else "smem"), (d, nq))
    return out


def test_dim_list_covers_every_residual_class():
    cov = coverage()
    want = []
    for kernel in SWEPT:
        v = KERNEL_V[kernel]
        want.append(("fp32", kernel, v, "dim<8", None))
        for rc in ("r0", "r1-15", "r16", "r17-31"):
            for nc in ("n0", "n<U", "n%U=0", "n>U,n%U!=0"):
                if (rc, nc) != ("r0", "n0") and not (nc == "n<U" and unroll(v) == 1):
                    want.append(("fp32", kernel, v, rc, nc))
    for name, width in (("int8/uint8", I8_VEC), ("fp16/bf16", H16_VEC)):
        for c in ("nvec<32", "nvec=32", "nvec>32,%32!=0"):
            for tail in ("tail", "no tail"):
                want.append((name, c, tail))
    for vtype in (F32, F16, BF16, I8, U8):
        for metric in (L2, IP, COS):
            for labels in ("rows", "labels"):
                for where in ("smem", "L1"):
                    want.append((TNAME[vtype], MNAME[metric], labels, where))
    missing = [w for w in want if w not in cov]
    assert not missing, missing
    for w in sorted(cov, key=str):
        print(w, "->", cov[w])
    # the route's rescoring: the classes their dims reach (every residual class, below / at / past U chunks)
    for kernel in PARTIAL:
        got = {c[3:] for c in cov if c[1] == kernel}
        assert {"r0", "r1-15", "r16", "r17-31"} <= {c[0] for c in got}, (kernel, got)
        assert {"n<U", "n>U,n%U!=0"} <= {c[1] for c in got}, (kernel, got)
    # the worked examples of the classes
    assert [f32_class(d, 4)[1] for d in (288, 300, 304, 311)] == ["n>U,n%U!=0"] * 4
    assert [f32_class(d, 4)[0] for d in (288, 300, 304, 311)] == ["r0", "r1-15", "r16", "r17-31"]
    assert queries_through_l1(F32, L2, 771, 64, 10) and not queries_through_l1(F32, L2, 771, 9, 10)
    assert queries_through_l1(F16, IP, 771, 64, 10) and not queries_through_l1(F16, IP, 768, 64, 10)
    assert queries_through_l1(I8, L2, 1553, 64, 10) and not queries_through_l1(I8, L2, 1536, 64, 10)
    assert queries_through_l1(I8, COS, 1533, 64, 10) and not queries_through_l1(I8, COS, 1532, 64, 10)
    # label-aware lists: at k = 128 the 64 KB more of labels do not move the L1 boundary (kMaxQuerySmem binds first)
    assert queries_through_l1(F32, L2, 385, 64, 128, True) and not queries_through_l1(F32, L2, 384, 64, 128, True)


# ------------------------------------------------------------------------------------------------------------------
# the plain reference of the 8-bit distances, and the fp32 restatement against the reference's code
# ------------------------------------------------------------------------------------------------------------------
def int_scores(X, y, metric, vtype, dim):
    """The reference's int8 / uint8 distance of every stored row X [n, stored bytes] to the stored query y: the exact
    integer dot product or squared L2 (int64), then its float expression (IP.cpp / L2.cpp): L2 float(e), IP float(1 - dot),
    cosine 1 - float(dot) / (nr * nq) in fp32 with the norms stored after the dim payload bytes."""
    t = np.int8 if vtype == I8 else np.uint8
    a = np.ascontiguousarray(X[:, :dim]).view(t).astype(np.int64)
    b = np.ascontiguousarray(y[:dim]).view(t).astype(np.int64)
    if metric == L2:
        d = a - b
        return np.einsum("ij,ij->i", d, d).astype(np.float32)
    dot = a @ b
    if metric == IP:
        return (1 - dot).astype(np.float32)
    nr = np.ascontiguousarray(X[:, dim:dim + 4]).view(np.float32)[:, 0]
    nq = np.ascontiguousarray(y[dim:dim + 4]).view(np.float32)[0]
    with np.errstate(invalid="ignore", divide="ignore"):  # an all-zero uint8 row: norm 0, 0 / 0 = NaN as in the reference
        return (np.float32(1.0) - dot.astype(np.float32) / (nr * nq)).astype(np.float32)


def _int_rows(vtype, metric, n, dim, seed):
    """Stored 8-bit rows (with the cosine norm appended the way orc_normalize stores it) and stored queries; extremes
    included (-128 / 127 / 0 / 255) so that the widest products and sums occur."""
    rows = ol.synth_rows(vtype, seed, 0, n, dim)
    lo, hi = (-128, 127) if vtype == I8 else (0, 255)
    rows[0] = lo
    rows[1] = hi
    rows[2, ::2] = lo
    rows[2, 1::2] = hi
    size = ol.port().orc_stored_size(vtype, dim, metric)
    out = np.zeros((n, size), dtype=np.uint8)
    out[:, :dim] = rows.view(np.uint8)
    if metric == COS:
        for r in out:
            ol.port().orc_normalize(ol._p(r), dim, vtype)
    return out


@pytest.mark.parametrize("metric", [L2, IP, COS])
@pytest.mark.parametrize("vtype", [I8, U8])
def test_plain_int_reference_equals_the_c_restatement(vtype, metric):
    L = ol.port()
    for dim in DIMS:
        X = _int_rows(vtype, metric, 40, dim, 7 + dim)
        for j in (0, 1, 2, 5):
            got = int_scores(X, X[j], metric, vtype, dim)
            want = np.array([L.orc_distance(vtype, metric, dim, ol._p(X[i]), ol._p(X[j]), ol.TIER_AVX512) for i in range(len(X))],
                            dtype=np.float32)
            assert got.tobytes() == want.tobytes(), (dim, j, np.flatnonzero(got != want)[:5])


def f32_scores(X, Y, metric, dim):
    """[nq, n] float32: the reference's AVX-512-tier fp32 distance (the C restatement, pinned to the reference's compiled
    code by test_oracle_vecsim.py) of every stored row to every stored query.  Cosine: the rows and queries are stored
    normalised, and the fp32 cosine distance is the inner-product one (1 - dot) of the stored vectors."""
    n, nq = X.shape[0], Y.shape[0]
    mt = L2 if metric == L2 else IP
    lab = np.zeros((nq, n), dtype=np.uint64)
    sc = np.zeros((nq, n), dtype=np.float32)
    cnt = np.zeros(nq, dtype=np.uint64)
    X, Y = np.ascontiguousarray(X, dtype=np.float32), np.ascontiguousarray(Y, dtype=np.float32)
    ol.port().orc_scan_topk_chunk(F32, mt, ol.TIER_AVX512, dim, ol._p(X), X.strides[0], n, 0, ol._p(Y), Y.strides[0], nq, n, 8,
                                  ol._p(lab), ol._p(sc), ol._p(cnt))
    assert (cnt == n).all()
    out = np.empty((nq, n), dtype=np.float32)
    for i in range(nq):
        out[i, lab[i].astype(np.int64)] = sc[i]
    return out


@pytest.mark.parametrize("metric", [L2, IP])
def test_fp32_restatement_over_the_dim_list(metric):
    """f32_scores (the batched C restatement) equals orc_distance row by row; and both equal the reference's compiled
    fp32 kernel where oracle/_ref is built and the host has AVX-512F."""
    L = ol.port()
    ref = ol.ref_vecsim() if ol.host_has_avx512f() else None
    for dim in DIMS:
        X = ol.synth_rows(F32, 11 + dim, 0, 30, dim)
        Y = ol.synth_rows(F32, 12 + dim, 0, 3, dim)
        S = f32_scores(X, Y, metric, dim)
        for j in range(len(Y)):
            one = np.array([L.orc_distance(F32, metric, dim, ol._p(X[i]), ol._p(Y[j]), ol.TIER_AVX512) for i in range(len(X))],
                           dtype=np.float32)
            assert one.tobytes() == S[j].tobytes(), (dim, j)
            if ref is not None:
                r = np.array([ref.Ref_Distance(F32, metric, dim, ol._p(X[i]), ol._p(Y[j])) for i in range(len(X))], dtype=np.float32)
                assert r.tobytes() == one.tobytes(), (dim, j)


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _vs():
    from redisearch_b200 import vecsim

    return vecsim


def _nonzero(x):
    """No all-zero 8-bit vector: its cosine norm is 0 and every distance to it NaN, which no selection orders."""
    if x.dtype in (np.int8, np.uint8):
        x[~x.any(axis=-1), 0] = 1
    return x


def _corpus(vtype, n, dim, seed):
    rows = _nonzero(ol.synth_rows(vtype, seed, 0, n, dim))
    rows[n // 2:n // 2 + 40] = rows[10:50]  # exact duplicates: ties that must resolve by label
    return rows


def _read_stored(g, n):
    size = g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)  # == the stored row bytes
    out = np.empty((n, size), dtype=np.uint8)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, out.ctypes.data) == 0
    return out


def reference_scores(g, vtype, metric, qs, n):
    """S [nq, n + 1] float32, indexed by label (= row + 1; NaN at 0): the reference's score of every stored row to the
    library's stored form of every query."""
    dim = g.dim
    X = _read_stored(g, n)
    Q = stored_queries(g, qs)
    if vtype == F32:
        S = f32_scores(X.view(np.float32), Q[:, :4 * dim].view(np.float32), metric, dim)
    else:
        S = np.stack([int_scores(X, Q[i], metric, vtype, dim) for i in range(len(qs))])
    return np.hstack([np.full((len(qs), 1), np.nan, dtype=np.float32), S])


def _batch_rows(bl, bs, i):
    h = int((bl[i] != SIZE_MAX).sum())
    return bl[i, :h].astype(np.int64), bs[i, :h]


def _single_query_paths(g, q, qb, S, n, tag):
    vs = _vs()
    want_l, want_s = selection(S, n)
    it = g.batch_iterator(q)  # scan_scores_kernel
    got_l, got_s = [], []
    while it.has_next():
        ids, sc, code = it.next(347, vs.BY_SCORE)
        assert code == 0
        if not len(ids):
            break
        got_l += ids.tolist()
        got_s += sc.tolist()
    it.free()
    assert_same_bits(got_l, got_s, want_l, want_s, (tag, "batch iterator"))
    for k in BATCH_K:  # scan_topk 4x1 (k <= 128) and scan_scores + select (k > 128)
        gi, gs, code = g.topk(q, k)
        assert code == 0
        assert_same_bits(gi, gs, *selection(S, k), (tag, k, "TopKQuery"))
    for pos in (0, 9, 37):  # range: scan_scores_kernel
        radius = max(0.0, float(want_s[min(pos, n - 1)]))
        ri, rs, code = g.range(q, radius)
        assert code == 0
        inside = ~np.isnan(S) & (S <= np.float32(radius))
        assert sorted(ri.tolist()) == np.flatnonzero(inside).tolist(), (tag, pos, "range")
        assert rs.astype(np.float32).tobytes() == S[ri].tobytes(), (tag, pos, "range")
    for allowed in (None, np.arange(n + 1) % 3 == 1):  # gather_kernel
        ids = np.arange(1, n + 1, dtype=np.uint32) if allowed is None else np.flatnonzero(allowed).astype(np.uint32)
        fl, fs, rc = g.topk_filtered(q, 10, ids)
        assert rc == 0
        assert_same_bits(fl, fs, *selection(S, 10, allowed), (tag, "TopKFiltered"))
    labs = np.array([11, 12, n // 2 + 11, n // 2 + 12, 1, 2, 3, n] + want_l[:5].tolist(), dtype=np.uint64)
    d = np.array([g.distance_from(int(lab), qb) for lab in labs], dtype=np.float32)
    assert d.tobytes() == S[labs.astype(np.int64)].tobytes(), (tag, "GetDistanceFrom")
    assert np.isnan(g.distance_from(n + 7, qb))
    a = g.adhoc_distances(q, np.arange(1, n + 1, dtype=np.uint64)).astype(np.float32)
    assert a.tobytes() == S[1:].tobytes(), (tag, "ad-hoc")


def _batched_paths(g, Q, S, tag):
    """Exact-scan batches (SetCoarseMode(0)): scan_topk 4x8 with the queries in shared memory or through L1, and
    scan_scores_wide 4x8 for k > 128; then the range batch."""
    vs = _vs()
    L = vs.lib()
    L.VecSimB200_SetCoarseMode(0)
    try:
        for nq in BATCH_NQ:
            for k in BATCH_K:
                bl, bs, rc = g.topk_batch(Q[:nq], k)
                assert rc == 0 and L.VecSimB200_LastBatchPath(g.h) == 0, (tag, nq, k)
                for i in range(nq):
                    assert_same_bits(*_batch_rows(bl, bs, i), *selection(S[i], k), (tag, nq, k, i, "TopKQueryBatch"))
        nq = 9
        radii = np.array([max(0.0, float(selection(S[i], 20)[1][-1])) for i in range(nq)])
        replies, rc, flags = g.range_batch(Q[:nq], radii)
        assert rc == 0 and not flags.any()
        for i, (ri, rs, code) in enumerate(replies):
            inside = ~np.isnan(S[i]) & (S[i] <= np.float32(radii[i]))
            assert code == 0 and sorted(ri.tolist()) == np.flatnonzero(inside).tolist(), (tag, i, "RangeQueryBatch")
            assert rs.astype(np.float32).tobytes() == S[i][ri].tobytes(), (tag, i, "RangeQueryBatch")
    finally:
        L.VecSimB200_SetCoarseMode(-1)


def _ragged_filters(rng, n, deleted):
    """0, 1, a few (an absent id and a deleted one among them) and thousands of ids (past the index included)."""
    few = np.array(sorted({3, 11, n // 2 + 11, deleted[0], n + 4} | set(rng.choice(np.arange(1, n + 1), 6).tolist())), dtype=np.uint32)
    many = np.arange(1, n + 2500, dtype=np.uint32)
    third = np.arange(1, n + 1, 3, dtype=np.uint32)
    return [np.zeros(0, dtype=np.uint32), np.array([n // 2 + 12], dtype=np.uint32), few, many, third, np.array([deleted[1]], dtype=np.uint32)]


def _check_ragged(g, qs, S_of, filters, ks, tag):
    """gather_ragged_kernel: every query's row equals the selection over the allowed labels of S_of[i] (NaN = absent)."""
    for k in ks:
        labels, scores, counts = ragged_batch(g, qs, k, filters)
        for i, f in enumerate(filters):
            allowed = np.zeros(len(S_of[i]), dtype=bool)
            f = f[f < len(allowed)].astype(np.int64)
            allowed[f] = True
            wl, ws = selection(S_of[i], k, allowed)
            c = int(counts[i])
            assert c == len(wl), (tag, k, i, c, len(wl))
            assert_same_bits(labels[i, :c], scores[i, :c], wl, ws, (tag, k, i, "TopKFilteredBatchDevice"))
            assert (labels[i, c:] == -1).all() and np.isnan(scores[i, c:]).all(), (tag, k, i)


# ------------------------------------------------------------------------------------------------------------------
# GPU: fp32 / int8 / uint8 single-value indexes, every CUDA-core path, every dim of the list
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP, COS])
@pytest.mark.parametrize("vtype", [F32, I8, U8])
def test_every_cuda_core_path_bit_equal_over_the_dim_list(vtype, metric):
    vs = _vs()
    n = 1200
    for dim in DIMS:
        rows = _corpus(vtype, n, dim, 700 + dim)
        g = vs.VecSimIndex(VT[vtype], dim, MT[metric])
        assert g.add_many(rows, label0=1) == n
        qs = _nonzero(ol.synth_rows(vtype, 800 + dim, 0, max(BATCH_NQ), dim))
        qs[1] = rows[13]  # its best rows include the tied duplicate pair 14 / n // 2 + 14
        qs[2] = rows[0]
        S = reference_scores(g, vtype, metric, qs, n)
        Q = stored_queries(g, qs)
        size = g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)
        for j in range(3):
            _single_query_paths(g, qs[j], Q[j, :size], S[j], n, (dim, j))
        _batched_paths(g, qs, S, (dim,))
        # the ragged device batch, after deletions (swap-delete moves the last rows into the holes)
        rng = np.random.default_rng(dim)
        deleted = [7, n - 3, 600]
        for lab in deleted:
            assert g.delete(lab) == 1
        S_del = S[:8].copy()
        S_del[:, deleted] = np.nan
        filters = _ragged_filters(rng, n, deleted)
        nf = len(filters)
        _check_ragged(g, qs[:nf], S_del[:nf], filters, (1, 10, 129), (dim, "ragged"))
        g.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU: fp16 / bf16 single-value — the paths test_cuda_core_paths_over_dim_residuals does not reach
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP, COS])
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_half_precision_ragged_batch_and_queries_through_l1(vtype, metric):
    vs = _vs()
    L = vs.lib()
    n = 1200
    for dim in HALF_DIMS:
        rows = _corpus(vtype, n, dim, 900 + dim)
        g = vs.VecSimIndex(VT[vtype], dim, MT[metric])
        assert g.add_many(rows, label0=1) == n
        qs = ol.synth_rows(vtype, 950 + dim, 0, 64, dim)
        qs[1] = rows[13]
        X = decode16(stored_rows(g, n), vtype)
        S = np.stack([single_scan_scores(g, q, n) for q in qs])
        E, B = [], []
        for q in qs:
            y = decode16(stored_query(g, q).view(np.uint16)[:dim], vtype)
            e, mag = exact_distances(X, y, metric)
            E.append(np.concatenate([[np.nan], e]))
            B.append(np.concatenate([[np.nan], bound_cuda_core(e, mag, dim)]))
        r = np.abs(S[:, 1:].astype(np.float64) - np.stack(E)[:, 1:]) / np.stack(B)[:, 1:]
        assert (r <= 1.0).all(), (dim, r.max())
        L.VecSimB200_SetCoarseMode(0)
        try:
            for k in (10, 128):
                # by the restated rule (the instantiation itself is not observable): queries through L1 at 771 and 1553
                assert queries_through_l1(vtype, metric, dim, 64, k) == (dim >= 771)
                bl, bs, rc = g.topk_batch(qs, k)
                assert rc == 0 and L.VecSimB200_LastBatchPath(g.h) == 0
                for i in range(64):
                    gl, gs = _batch_rows(bl, bs, i)
                    assert_same_bits(gl, gs, *selection(S[i], k), (dim, k, i, "TopKQueryBatch"))
                    if i < 4:
                        check_answer(gl, gs, E[i], B[i], k)
        finally:
            L.VecSimB200_SetCoarseMode(-1)
        deleted = [7, n - 3]
        for lab in deleted:
            assert g.delete(lab) == 1
        S_del = S[:6].copy()
        S_del[:, deleted] = np.nan
        filters = _ragged_filters(np.random.default_rng(dim), n, deleted)
        _check_ragged(g, qs[:len(filters)], S_del[:len(filters)], filters, (10, 129), (dim, "ragged"))
        g.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU: multi-value indexes, all five types
# ------------------------------------------------------------------------------------------------------------------
def _multi_expected(row_scores, row_labels, n_labels):
    """From the per-row scores [nq, n] of a multi-value index (rows in insertion order = row ids): S [nq, n_labels + 1], the
    reference's fold of each label's rows (brute_force_multi.h:234-238; no NaN here, so the minimum), and R [nq, n_labels + 1],
    the lowest row id among the label's rows that reach S.  The device's label-aware scans select on (score, row) composites,
    so among labels tied exactly at the k-th score the ones with the lower best row are kept, where the reference keeps the
    lower labels (DESIGN.md §3.2, the documented tie deviation); replies are in (score, label) order either way.  Filtered
    KNN and the ragged batch select by (score, docId), like the reference."""
    nq, n = row_scores.shape
    S = np.full((nq, n_labels + 1), np.nan, dtype=np.float32)
    R = np.full((nq, n_labels + 1), n, dtype=np.int64)
    rows = np.arange(n)
    for i in range(nq):
        order = np.lexsort((rows, row_scores[i], row_labels))
        first = np.ones(n, dtype=bool)
        first[1:] = row_labels[order][1:] != row_labels[order][:-1]
        S[i, row_labels[order][first]] = row_scores[i][order][first]
        R[i, row_labels[order][first]] = order[first]
    return S, R


def scan_selection(S, R, k):
    """(labels, score bits) of the device's label-aware scans: the k labels first in (score, best row) order, replied in
    (score, label) order."""
    labels = np.flatnonzero(~np.isnan(S))
    kept = labels[np.lexsort((R[labels], S[labels]))[:k]]
    kept = kept[np.lexsort((kept, S[kept]))]
    return kept, S[kept]


def _check_scan_answer(gl, gs, S, R, k, what):
    """Bit-equal to the device's documented order; the same score bits as the reference's (score, label) selection, and the
    same labels wherever the k-th score is not tied across the boundary."""
    assert_same_bits(gl, gs, *scan_selection(S, R, k), what)
    rl, rs = selection(S, k)
    assert np.asarray(gs, dtype=np.float32).tobytes() == rs.tobytes(), what
    tied = rs == rs[-1] if len(rs) else rs.astype(bool)
    assert set(np.asarray(gl)[~tied].tolist()) == set(rl[~tied].tolist()), what


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP, COS])
@pytest.mark.parametrize("vtype", [F32, I8, U8, F16, BF16])
def test_multi_value_cuda_core_paths_over_the_dim_list(vtype, metric):
    """Three rows per label, scattered, exact duplicate rows under different labels: the label-aware scan_topk (TopKQuery,
    TopKQueryBatch on the exact scan with the queries in shared memory or through L1), gather_min (TopKFiltered),
    gather_ragged<MULTI> (the device filtered batch) and GetDistanceFrom.  fp32 / int8 / uint8: per-row scores from the
    reference's arithmetic, the fold pinned to PortIndex(multi=True).  fp16 / bf16: per-row scores of the single-value
    index over the same rows (bit-equal on every CUDA-core path), reference_fold over them, within B_cc of fp64."""
    vs = _vs()
    L = vs.lib()
    n_labels = 400
    n = 3 * n_labels
    half = vtype in (F16, BF16)
    for dim in (HALF_DIMS if half else DIMS):
        rng = np.random.default_rng(1000 + dim)
        rows = _corpus(vtype, n, dim, 1100 + dim)
        row_labels = (np.arange(n, dtype=np.int64) // 3 + 1)[rng.permutation(n)]
        g = vs.VecSimIndex(VT[vtype], dim, MT[metric], multi=True)
        assert g.add_many(rows, labels=row_labels.astype(np.uint64)) == n
        qs = _nonzero(ol.synth_rows(vtype, 1200 + dim, 0, max(MULTI_NQ), dim))
        qs[1] = rows[13]
        Q = stored_queries(g, qs)
        size = g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)
        if half:
            single = vs.VecSimIndex(VT[vtype], dim, MT[metric])
            assert single.add_many(rows, label0=1) == n
            row_scores = np.stack([single_scan_scores(single, q, n)[1:] for q in qs])
            X = decode16(stored_rows(single, n), vtype)
            single.close()
        else:
            row_scores = reference_scores(g, vtype, metric, qs, n)[:, 1:]
        S, R = _multi_expected(row_scores, row_labels, n_labels)
        bounds = []
        if not half:
            p = ol.PortIndex(vtype, dim, metric, multi=True, tier=ol.TIER_AVX512)
            for r, lab in zip(rows, row_labels.tolist()):
                p.add(r, lab)
        for j in range(2):
            if half:  # reference_fold in insertion order, and B_cc of the fp64 distance
                for lab in (1, 2, row_labels[13], n_labels):
                    assert reference_fold(row_scores[j][row_labels == lab]).tobytes() == S[j, lab].tobytes()
                y = decode16(stored_query(g, qs[j]).view(np.uint16)[:dim], vtype)
                e, mag = exact_distances(X, y, metric)
                bounds.append(per_label(e, bound_cuda_core(e, mag, dim), row_labels, n_labels + 1))
            else:  # the fold equals the reference's multi-value getDistanceFrom
                want = np.array([p.distance_from(lab, Q[j]) for lab in range(1, n_labels + 1)], dtype=np.float32)
                assert want.tobytes() == S[j, 1:].tobytes(), (dim, j, "fold")
        for j in range(2):
            for k in (1, 10, 128):  # scan_topk 4x1, label-aware lists
                gi, gs, code = g.topk(qs[j], k)
                assert code == 0
                _check_scan_answer(gi, gs, S[j], R[j], k, (dim, j, k, "TopKQuery multi"))
                if half:
                    check_answer(gi, gs, bounds[j][0], bounds[j][1], k, tie_order=False)
            for allowed in (None, np.arange(n_labels + 1) % 3 == 1):  # gather_min_kernel
                ids = np.arange(1, n_labels + 1, dtype=np.uint32) if allowed is None else np.flatnonzero(allowed).astype(np.uint32)
                for k in (10, 128):
                    fl, fs, rc = g.topk_filtered(qs[j], k, ids)
                    assert rc == 0
                    assert_same_bits(fl, fs, *selection(S[j], k, allowed), (dim, j, k, "TopKFiltered multi"))
            d = np.array([g.distance_from(lab, Q[j, :size]) for lab in range(1, n_labels + 1)], dtype=np.float32)
            assert d.tobytes() == S[j, 1:].tobytes(), (dim, j, "GetDistanceFrom multi")
        L.VecSimB200_SetCoarseMode(0)
        try:  # scan_topk 4x8 with label-aware lists: queries in shared memory, or through L1 at the wide dims
            for nq, k in ((9, 10), (64, 10), (64, 128)):
                bl, bs, rc = g.topk_batch(qs[:nq], k)
                assert rc == 0 and L.VecSimB200_LastBatchPath(g.h) == 0
                for i in range(nq):
                    _check_scan_answer(*_batch_rows(bl, bs, i), S[i], R[i], k, (dim, nq, k, i, "TopKQueryBatch multi"))
        finally:
            L.VecSimB200_SetCoarseMode(-1)
        filters = [np.zeros(0, dtype=np.uint32), np.array([5], dtype=np.uint32),
                   np.array([2, 9, 77, n_labels + 3], dtype=np.uint32), np.arange(1, n_labels + 900, dtype=np.uint32)]
        _check_ragged(g, qs[:4], S[:4], filters, (1, 10, 129), (dim, "ragged multi"))
        g.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU: the fp32 tensor-core route's exact rescoring (refine_kernel, range_refine_kernel)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [COS, L2])
def test_tensor_core_rescoring_bit_equal_over_residual_classes(metric):
    vs = _vs()
    L = vs.lib()
    n, nq, k = 65_536, 16, 10
    L.VecSimB200_SetCoarseMode(1)
    try:
        for dim in (40, 56, 72, 288, 304, 1000):
            rows = ol.synth_rows(F32, 1300 + dim, 0, n, dim)
            g = vs.VecSimIndex(VT[F32], dim, MT[metric])
            assert g.add_many(rows, label0=1) == n
            p = ol.PortIndex(F32, dim, metric, tier=ol.TIER_AVX512)
            p.add_many(rows, 1)
            qs = ol.synth_rows(F32, 1400 + dim, 0, nq, dim)
            # the device batch keeps per-query flags: 1 / 2 = answered by the route (refine_kernel's rescoring), 0 = the exact scan
            dl, ds = device_batch(g, stored_queries(g, qs), k)
            assert L.VecSimB200_LastBatchPath(g.h) == 1, (dim, "the batch did not take the route")
            f = flags_of(g, nq)
            assert f is not None and ((f == 1) | (f == 2)).sum() >= nq // 2, (dim, f)
            bl, bs, rc = g.topk_batch(qs, k)
            assert rc == 0 and L.VecSimB200_LastBatchPath(g.h) == 1
            assert (bl.astype(np.int64) == dl).all() and bs.astype(np.float32).tobytes() == ds.astype(np.float32).tobytes(), dim
            for i in range(nq):
                if f[i] == 0 and i % 2:
                    continue
                pi, ps = p.topk(qs[i], k)
                assert_same_bits(dl[i], ds[i], pi, ps, (dim, i, int(f[i]), "TopKQueryBatchDevice route"))
            radii = bs[:, k - 1].astype(np.float32).astype(np.float64)
            replies, rc, rflags = g.range_batch(qs, radii)
            assert rc == 0 and rflags.any(), (dim, rflags)
            for i in range(0, nq, 2):
                pi, ps = p.range(qs[i], float(radii[i]))
                ri, rs, code = replies[i]
                assert code == 0
                assert_same_bits(ri, rs, pi, ps, (dim, i, "RangeQueryBatch route"))
            g.close()
    finally:
        L.VecSimB200_SetCoarseMode(-1)
