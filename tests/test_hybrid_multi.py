"""GPU: filtered KNN on multi-value indexes (a docId owns several rows) — VecSimB200_TopKFiltered, VecSimB200_TopKFilteredBatch and
VecSimB200_HybridTopK in every mode — against the reference's ad-hoc hybrid loop (src/iterators/hybrid_reader.c:289-335) driven by
the reference's own getDistanceFrom_Unsafe with multi=True (brute_force_multi.h:224-241: dist = +inf, then
dist = (dist < d) ? dist : d over the label's rows in insertion order).  The oracle is the reference's compiled VecSim when
oracle/_ref is built, else the C restatement.  Ids and fp32 score bits must be equal for fp32 and the 8-bit types; fp16 / bf16 are
held to the 1e-2 bar.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from test_hybrid_filtered import _oracle_adhoc
from test_vecsim_parity import assert_same

pytestmark = pytest.mark.gpu


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


def _oracle(vtype, dim, metric):
    if ol.ref_vecsim() is not None:
        return ol.RefIndex(vtype, dim, metric, multi=True)
    return ol.PortIndex(vtype, dim, metric, multi=True, tier=ol.TIER_AVX512)


def _query_blob(g, q, dim, vtype, metric):
    """The query as the reference's loop hands it to getDistanceFrom_Unsafe: normalised by the caller for cosine
    (hybrid_reader.c:296-305)."""
    vs = _vs()
    qb = np.zeros(g.L.VecSimParams_GetQueryBlobSize(vtype, dim, metric), dtype=np.uint8)
    qb[: q.nbytes] = q.view(np.uint8)
    if metric == ol.COS:
        vs.normalize(qb, dim, vtype)
    return qb


def _uneven_labels(rng, n):
    """Per-row docIds for n rows: 1..60 rows per label (most labels small, a few large), spaced by 2, rows scattered."""
    counts = []
    while sum(counts) < n:
        counts.append(int(rng.integers(30, 61)) if rng.random() < 0.08 else int(rng.integers(1, 6)))
    counts[-1] -= sum(counts) - n
    if counts[-1] == 0:
        counts.pop()
    lab = np.repeat(1 + 2 * np.arange(len(counts), dtype=np.uint64), counts)
    return lab[rng.permutation(n)], 1 + 2 * np.arange(len(counts), dtype=np.uint64)


def _add_both(g, o, rows, labels):
    assert g.add_many(rows, labels=labels) == len(rows)
    for r, lab in zip(rows, labels.tolist()):
        o.add(r, lab)


CASES = [(ol.F32, ol.COS), (ol.F32, ol.L2), (ol.F32, ol.IP), (ol.I8, ol.COS), (ol.U8, ol.IP), (ol.F16, ol.IP), (ol.BF16, ol.COS)]


@pytest.mark.parametrize("dim", [64, 100])
@pytest.mark.parametrize("vtype,metric", CASES)
def test_topk_filtered_on_a_multi_value_index_matches_the_adhoc_loop(vtype, metric, dim):
    import torch

    vs = _vs()
    n, k = 12_000, 10
    rng = np.random.default_rng(1000 * vtype + 10 * metric + dim)
    rows = ol.synth_rows(vtype, 42 + dim, 0, n, dim)
    labels, owners = _uneven_labels(rng, n)
    g = vs.VecSimIndex(vtype, dim, metric, multi=True)
    o = _oracle(vtype, dim, metric)
    _add_both(g, o, rows, labels)
    top = int(owners[-1])
    exact = vtype in (ol.F32, ol.I8, ol.U8)
    qs = ol.synth_rows(vtype, 43 + dim, 0, 3, dim)

    def check(stage, q):
        qb = _query_blob(g, q, dim, vtype, metric)
        for m in (0, 3, 500, 3000):
            # even ids (never labels), deleted labels and ids past the end included
            doc_ids = np.sort(rng.choice(np.arange(1, top + 400), m, replace=False)).astype(np.uint32)
            exp = _oracle_adhoc(o, qb, doc_ids, k)
            ei = np.array([d for _, d in exp], dtype=np.int64)
            es = np.array([s for s, _ in exp], dtype=np.float32)
            labs, scores, rc = g.topk_filtered(q, k, doc_ids)
            assert rc == 0, (stage, m)
            assert_same(labs.astype(np.int64), scores, ei, es, exact, metric)
            if m >= 500:  # the same filter as a device-resident list
                d_ids = torch.from_numpy(doc_ids).cuda()
                dl, dsc, rc = g.topk_filtered(q, k, d_ids.data_ptr(), n=m)
                assert rc == 0 and dl.tolist() == labs.tolist() and dsc.tobytes() == scores.tobytes(), (stage, m)

    check("fresh", qs[0])
    # whole labels deleted: their rows leave by swap-delete, which moves rows of surviving labels into the holes
    gone = rng.choice(owners, len(owners) // 5, replace=False)
    for lab in gone.tolist():
        assert g.delete(int(lab)) > 0
        o.delete(int(lab))
    check("after deletes", qs[1])
    # rows added to labels that still exist, after the deletes: the label -> rows table has to be rebuilt
    alive = np.setdiff1d(owners, gone)
    more = ol.synth_rows(vtype, 44 + dim, 0, 600, dim)
    _add_both(g, o, more, rng.choice(alive, 600))
    check("after re-adds", qs[2])


def test_the_fold_keeps_the_reference_order_over_nan_rows():
    """getDistanceFrom_Unsafe folds with dist = (dist < d) ? dist : d: a NaN row resets dist to NaN and the next row replaces it.
    Label 7's NaN row is its last one -> NaN, the docId is skipped; label 9's NaN row is its first one -> forgotten.  A plain min
    (or fminf) would answer label 7 too."""
    vs = _vs()
    dim, k = 32, 20
    rng = np.random.default_rng(5)
    rows, labels = [], []
    for lab in range(1, 21):  # docIds 1..20, two rows each, three for 7 and 9
        nr = 3 if lab in (7, 9) else 2
        for j in range(nr):
            r = rng.standard_normal(dim).astype(np.float32)
            if (lab == 7 and j == nr - 1) or (lab == 9 and j == 0):
                r[3] = np.nan  # one NaN component: the row's L2 distance is NaN
            rows.append(r)
            labels.append(lab)
    rows, labels = np.stack(rows), np.array(labels, dtype=np.uint64)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2, multi=True)
    o = _oracle(ol.F32, dim, ol.L2)
    _add_both(g, o, rows, labels)
    q = rng.standard_normal(dim).astype(np.float32)
    doc_ids = np.arange(1, 21, dtype=np.uint32)
    labs, scores, rc = g.topk_filtered(q, k, doc_ids)
    assert rc == 0
    assert 7 not in labs.tolist() and 9 in labs.tolist()
    assert len(labs) == 19
    # label 9 scores as its good rows do; the index's own distance for them (both rows are non-NaN) is the reference's
    d9 = float(scores[labs.tolist().index(9)])
    assert np.float32(d9).tobytes() == np.float32(o.distance_from(9, q)).tobytes()
    if isinstance(o, ol.RefIndex):
        assert np.isnan(o.distance_from(7, q))
        exp = _oracle_adhoc(o, q, doc_ids, k)
        assert labs.tolist() == [d for _, d in exp]
        assert scores.astype(np.float32).tobytes() == np.array([s for s, _ in exp], dtype=np.float32).tobytes()


def test_batched_filtered_knn_on_a_multi_value_index_equals_the_single_calls():
    """VecSimB200_TopKFilteredBatch on a multi-value index, filters from II_IntersectBatch (device-resident), an empty filter and
    one smaller than k included: equal to the per-query calls and to the oracle's ad-hoc loop."""
    from redisearch_b200 import postings as ps

    vs = _vs()
    n, dim, k, nq = 40_000, 64, 10, 20
    rng = np.random.default_rng(21)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    lab = (np.arange(n, dtype=np.uint64) // 4 + 1)[rng.permutation(n)]  # 4 rows per docId, scattered
    n_labels = n // 4
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
    o = _oracle(ol.F32, dim, ol.COS)
    _add_both(g, o, rows, lab)
    for d in rng.choice(np.arange(1, n_labels + 1), 300, replace=False).tolist():  # deleted docIds stay in the filters
        g.delete(int(d))
        o.delete(int(d))
    sizes = [8_000, 6_000, 3_000, 400, 60, 5, 0]
    pool = [np.unique(rng.integers(1, n_labels + 50, s)).astype(np.uint64) for s in sizes]
    pls = [ps.PostingList.from_arrays(x) for x in pool]
    pairs = [(int(rng.integers(0, len(pool))), int(rng.integers(0, len(pool)))) for _ in range(nq)]
    pairs[0], pairs[1] = (0, 6), (4, 5)  # an empty filter, a filter smaller than k
    P, L = ps.lib(), vs.lib()
    arrays = [(C.c_void_p * 2)(pls[a].h, pls[b].h) for a, b in pairs]
    lists_pp = (C.c_void_p * nq)(*[C.cast(a, C.c_void_p) for a in arrays])
    n_lists = (C.c_size_t * nq)(*([2] * nq))
    rs_out = (C.c_void_p * nq)()
    assert P.II_IntersectBatch(nq, lists_pp, n_lists, rs_out) == nq
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    q_ptrs = (C.c_void_p * nq)(*[qs[i].ctypes.data for i in range(nq)])
    id_ptrs, counts = (C.c_void_p * nq)(), (C.c_size_t * nq)()
    filters = []
    for i, (a, b) in enumerate(pairs):
        filt = np.intersect1d(pool[a], pool[b])
        filters.append(filt)
        assert P.II_ResultSet_Len(rs_out[i]) == len(filt)
        counts[i] = len(filt)
        id_ptrs[i] = P.II_ResultSet_DeviceDocIds(rs_out[i]) if len(filt) else None
    out_l = np.zeros((nq, k), dtype=np.uint64)
    out_s = np.zeros((nq, k), dtype=np.float64)
    out_c = (C.c_size_t * nq)()
    assert L.VecSimB200_TopKFilteredBatch(g.h, q_ptrs, nq, k, id_ptrs, counts, out_l.ctypes.data, out_s.ctypes.data, out_c) == 0
    for i in range(nq):
        qn = qs[i].copy()
        ol.port().orc_normalize(ol._p(qn), dim, ol.F32)
        exp = _oracle_adhoc(o, qn, filters[i], k)
        assert out_c[i] == len(exp), (i, pairs[i])
        assert out_l[i, :out_c[i]].tolist() == [d for _, d in exp]
        assert out_s[i, :out_c[i]].astype(np.float32).tobytes() == np.array([s for s, _ in exp], dtype=np.float32).tobytes()
        if len(filters[i]):
            labels, scores, rc = g.topk_filtered(qs[i], k, id_ptrs[i], n=len(filters[i]))
            assert rc == 0 and labels.tolist() == out_l[i, :out_c[i]].tolist()
            assert scores.astype(np.float32).tobytes() == out_s[i, :out_c[i]].astype(np.float32).tobytes()
        P.II_ResultSet_Free(rs_out[i])


@pytest.mark.parametrize("scenario", ["adhoc", "batches", "batches_then_adhoc", "few_matches"])
def test_hybrid_topk_on_a_multi_value_index_matches_the_reference_call_sequence(scenario):
    from redisearch_b200 import postings as ps
    from test_hybrid_state_machine import ADHOC, BATCHES, BATCHES_TO_ADHOC, oracle_hybrid

    if ol.ref_vecsim() is None:
        pytest.skip("the batches oracle drives the reference's batch iterator (oracle/_ref)")
    vs = _vs()
    n, dim, k = 60_000, 32, 10
    rng = np.random.default_rng(8)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    counts = rng.integers(1, 9, n)  # 1..8 rows per docId, scattered
    counts = counts[: int(np.searchsorted(np.cumsum(counts), n)) + 1]
    counts[-1] -= int(counts.sum()) - n
    n_labels = len(counts)
    lab = np.repeat(np.arange(1, n_labels + 1, dtype=np.uint64), counts)[rng.permutation(n)]
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
    ref = ol.RefIndex(ol.F32, dim, ol.COS, multi=True)
    _add_both(g, ref, rows, lab)
    q = ol.synth_rows(ol.F32, 43, 0, 1, dim)[0]
    qn = q.copy()
    ol.port().orc_normalize(ol._p(qn), dim, ol.F32)
    all_ids, _ = ref.topk(q, n_labels)  # every docId by distance
    assert len(all_ids) == n_labels
    if scenario == "adhoc":
        child_ids = np.sort(rng.choice(np.arange(1, n_labels + 1), n_labels // 20, replace=False))
    elif scenario == "batches":
        child_ids = np.sort(rng.choice(np.arange(1, n_labels + 1), n_labels // 2, replace=False))
    elif scenario == "batches_then_adhoc":
        child_ids = np.sort(all_ids[n_labels // 2:])  # the farthest half: batches keep finding nothing, the review switches
    else:
        child_ids = np.sort(rng.choice(np.arange(1, n_labels + 1), 4, replace=False))
    exp_mode, exp_iters, exp_ids, exp_sc = oracle_hybrid(ref, True, q, qn, k, child_ids)
    want = {"adhoc": ADHOC, "batches": BATCHES, "batches_then_adhoc": BATCHES_TO_ADHOC}.get(scenario)
    if want is not None:
        assert exp_mode == want, (scenario, exp_mode)

    pl = ps.PostingList.from_arrays(child_ids.astype(np.uint64))
    it = ps.union([pl]).into_iterator()
    qp = vs.VecSimQueryParams()
    labels = np.zeros(k, dtype=np.uint64)
    scores = np.zeros(k, dtype=np.float64)
    cnt, mode, iters = C.c_size_t(0), C.c_int(0), C.c_size_t(0)
    rc = vs.lib().VecSimB200_HybridTopK(g.h, q.ctypes.data, k, C.cast(it, C.c_void_p), C.byref(qp), labels.ctypes.data, scores.ctypes.data,
                                        C.byref(cnt), C.byref(mode), C.byref(iters))
    it.contents.Free(it)
    assert rc == 0
    assert mode.value == exp_mode, (scenario, mode.value, exp_mode)
    assert iters.value == exp_iters, (scenario, iters.value, exp_iters)
    assert labels[:cnt.value].tolist() == exp_ids, (scenario, labels[:cnt.value], exp_ids)
    assert scores[:cnt.value].astype(np.float32).tobytes() == exp_sc.tobytes()


def test_sparse_docids_still_refuse_the_filtered_query():
    """A docId at or beyond 2^32 leaves no dense label -> rows table: the filtered query answers -2, as on single-value indexes."""
    vs = _vs()
    dim = 16
    rows = ol.synth_rows(ol.F32, 42, 0, 6, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2, multi=True)
    assert g.add_many(rows, labels=np.array([1, 1, 2, 2, 2**32 + 5, 2**32 + 5], dtype=np.uint64)) == 6
    labs, _, rc = g.topk_filtered(rows[0], 3, np.array([1, 2], dtype=np.uint32))
    assert rc == -2 and len(labs) == 0
    assert g.delete(2**32 + 5) == 2  # dense again: served
    labs, scores, rc = g.topk_filtered(rows[0], 3, np.array([1, 2], dtype=np.uint32))
    assert rc == 0 and labs.tolist()[0] == 1 and scores[0] == 0.0
