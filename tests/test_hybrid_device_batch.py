"""Batches of filtered KNN queries on the device end to end: II_IntersectBatchDevice (the ANDs, no host wait) feeding
VecSimB200_TopKFilteredBatchDevice (ragged gather + segmented selection, counts read on the device).

Every query's row must be bit-equal to VecSimB200_TopKFiltered on the same filter (labels, order, score bits, count; -1 / NaN
tails).  fp32 / int8 / uint8 are also held to the reference's getDistanceFrom and its (distance, docId) order (the reference's
compiled VecSim when oracle/_ref is built, else the C restatement); fp16 / bf16 to the derived bounds of
test_half_precision_bounds.py.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from test_half_precision_bounds import bound_cuda_core, check_answer, decode16, exact_distances

pytestmark = pytest.mark.gpu

KS = [1, 10, 128, 129, 1000]
VARIANTS = [(ol.F32, ol.COS), (ol.F32, ol.IP), (ol.F32, ol.L2), (ol.F16, ol.IP), (ol.BF16, ol.L2), (ol.I8, ol.COS), (ol.U8, ol.L2)]


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


def _oracle(vtype, dim, metric, multi):
    if ol.ref_vecsim() is not None:
        return ol.RefIndex(vtype, dim, metric, multi=multi)
    return ol.PortIndex(vtype, dim, metric, multi=multi, tier=ol.TIER_AVX512)


def stored_queries(g, qs):
    """[nq, query_pitch] stored-form blobs: the library's own normaliser for cosine (int8 / uint8: norm appended)."""
    vs = _vs()
    size = g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)
    out = np.zeros((len(qs), g.query_pitch()), dtype=np.uint8)
    for i, q in enumerate(qs):
        b = np.zeros(size, dtype=np.uint8)
        b[: q.nbytes] = np.ascontiguousarray(q).view(np.uint8)
        if g.metric == vs.VecSimMetric_Cosine:
            vs.normalize(b, g.dim, g.vtype)
        out[i, :size] = b
    return out


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_batch(g, qs, k, filters, caps=None, exact_caps=False, stream=None):
    """One VecSimB200_TopKFilteredBatchDevice call; filters[i] = ascending uint32 docIds.  caps (default: the filter sizes) may
    exceed the counts, the device buffers then hold garbage up to the cap.  exact_caps: no count pointers.  Synchronises."""
    import torch

    bufs, cnts, ptrs, cps, cptrs = [], [], [], [], []
    for i, f in enumerate(filters):
        cap = len(f) if caps is None else caps[i]
        buf = np.full(max(cap, 1), 0xFFFFFFF0, dtype=np.uint32)  # past the count: ids the kernels must never read
        buf[: len(f)] = f
        bufs.append(_dev(buf.view(np.int32)))
        cnts.append(_dev(np.array([len(f)], dtype=np.int32)))
        ptrs.append(bufs[-1].data_ptr() if cap else None)
        cptrs.append(cnts[-1].data_ptr())
        cps.append(cap)
    qd = _dev(stored_queries(g, qs))
    labels, scores, counts, rc = g.topk_filtered_batch_device(qd, k, ptrs, cps, counts=None if exact_caps else cptrs, stream=stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy().astype(np.int64)


def assert_row_equals_filtered(g, q, k, filt, labels, scores, count, what):
    """labels / scores / count of one query against VecSimB200_TopKFiltered on the same filter; the tail -1 / NaN."""
    el, es, rc = g.topk_filtered(q, k, np.ascontiguousarray(filt, dtype=np.uint32))
    assert rc == 0, what
    n = len(el)
    assert count == n, (what, count, n)
    assert labels[:n].tolist() == el.astype(np.int64).tolist(), what
    assert scores[:n].tobytes() == es.astype(np.float32).tobytes(), what
    assert (labels[n:] == -1).all() and np.isnan(scores[n:]).all(), what
    return el.astype(np.int64), es.astype(np.float32)


def _oracle_row(o, qb, filt, k, dist_cache):
    """The reference's ad-hoc loop (hybrid_reader.c:289-335): getDistanceFrom per docId, NaN skipped, (distance, docId) order."""
    best = []
    for d in filt.tolist():
        if d not in dist_cache:
            dist_cache[d] = np.float32(o.distance_from(int(d), qb))
        s = dist_cache[d]
        if s == s:
            best.append((s, d))
    best.sort(key=lambda t: (t[0], t[1]))
    return best[:k]


def _corpus(vtype, metric, multi, rng):
    """A single-value index of 60K rows (docIds 1..60K) or a multi-value one of 30K rows over 10K docIds (3 each, scattered), with
    deleted docIds and, on float types of a multi-value index, a docId whose LAST row is NaN (-> NaN) and one whose FIRST is."""
    vs = _vs()
    dim = 48
    g = vs.VecSimIndex(vtype, dim, metric, multi=multi)
    o = _oracle(vtype, dim, metric, multi)
    deleted = set()
    if not multi:
        n = 60_000
        rows = ol.synth_rows(vtype, 42, 0, n, dim)
        assert g.add_many(rows, label0=1) == n
        o.add_many(rows, 1)
        top = n
    else:
        n = 30_000
        rows = ol.synth_rows(vtype, 42, 0, n, dim)
        labels = (np.arange(n, dtype=np.uint64) // 3 + 1)[rng.permutation(n)]
        assert g.add_many(rows, labels=labels) == n
        for r, lab in zip(rows, labels.tolist()):
            o.add(r, lab)
        top = n // 3
    for lab in rng.choice(np.arange(1, top + 1), top // 50, replace=False).tolist():
        g.delete(int(lab))
        o.delete(int(lab))
        deleted.add(lab)
    nan_labels = []
    if multi and vtype in (ol.F32, ol.F16, ol.BF16):
        good = ol.synth_rows(vtype, 44, 0, 2, dim)
        bad = good.copy()
        bad[:, 3] = np.float32("nan") if vtype == ol.F32 else np.uint16(0x7E00 if vtype == ol.F16 else 0x7FC0)
        last, first = top + 3, top + 5
        for lab, seq in ((last, (good[0], bad[0])), (first, (bad[1], good[1]))):
            for r in seq:
                assert g.add(r, lab) == 1
                o.add(r, lab)
        nan_labels = [last, first]
        top += 6
    return g, o, dim, top, nan_labels, rows, deleted


def _filters(rng, top, nan_labels):
    """Filter sizes 0, 1, fewer than k, some thousands and about 100K (ids past the index and deleted ids included)."""
    sizes = [0, 1, 5, 60, 3000, 100_000, 700, 2]
    out = []
    for s in sizes:
        hi = max(top + 50_000, s + 10)
        f = np.sort(rng.choice(np.arange(1, hi), s, replace=False)).astype(np.uint32)
        out.append(f)
    for lab in nan_labels:  # the NaN-last / NaN-first docIds in every non-empty filter
        out = [np.union1d(f, [lab]).astype(np.uint32) if len(f) else f for f in out]
    return out


@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
@pytest.mark.parametrize("vtype,metric", VARIANTS)
def test_device_batch_equals_topk_filtered_and_the_reference(vtype, metric, multi):
    rng = np.random.default_rng(100 * vtype + 10 * metric + int(multi))
    g, o, dim, top, nan_labels, rows, deleted = _corpus(vtype, metric, multi, rng)
    filters = _filters(rng, top, nan_labels)
    qs = ol.synth_rows(vtype, 43, 0, len(filters), dim)
    qst = stored_queries(g, qs)
    exact = vtype in (ol.F32, ol.I8, ol.U8)
    caches = [dict() for _ in filters]
    for k in KS:
        labels, scores, counts = device_batch(g, qs, k, filters)
        for i, f in enumerate(filters):
            what = (k, i, len(f))
            el, es = assert_row_equals_filtered(g, qs[i], k, f, labels[i], scores[i], counts[i], what)
            if nan_labels and len(f):
                assert nan_labels[0] not in el.tolist(), what  # a NaN in the last row makes the docId NaN
            qb = qst[i, : g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)]
            if exact and len(f) <= 5000:
                exp = _oracle_row(o, qb, f, k, caches[i])
                assert el.tolist() == [d for _, d in exp], what
                assert es.tobytes() == np.array([s for s, _ in exp], dtype=np.float32).tobytes(), what
            elif exact and k in (10, 1000):
                # the ~100K filter: every returned score is the reference's distance, in (distance, docId) order
                ref = np.array([np.float32(o.distance_from(int(d), qb)) for d in el.tolist()], dtype=np.float32)
                assert ref.tobytes() == es.tobytes(), what
                key = list(zip(es.tolist(), el.tolist()))
                assert key == sorted(key), what
            elif not exact and not multi and k in (10, 129) and len(f):
                # 16-bit: within the derived bound of the exact distance of the stored values (IP / L2 store the rows as given)
                e, mag = exact_distances(decode16(rows, vtype), decode16(qb.view(np.uint16)[:dim], vtype), metric)
                live = f[f <= top].astype(np.int64)
                live = live[~np.isin(live, list(deleted))]
                e_of, b_of = np.full(top + 1, np.nan), np.full(top + 1, np.nan)
                e_of[live], b_of[live] = e[live - 1], bound_cuda_core(e[live - 1], mag[live - 1], dim)
                check_answer(el, es.astype(np.float64), e_of, b_of, k, tie_order=True)


def _pool_lists(rng, n_top):
    from redisearch_b200 import postings as ps

    sizes = [40_000, 25_000, 9_000, 400, 60, 5, 0]
    pool = [np.unique(rng.integers(1, n_top + 50, s)).astype(np.uint64) for s in sizes]
    return pool, [ps.PostingList.from_arrays(x) for x in pool]


def _fp32_index(n=60_000, dim=64, multi=False):
    vs = _vs()
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=multi)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    assert g.add_many(rows, label0=1) == n
    return g, rows


@pytest.mark.parametrize("k", [10, 128])
def test_device_intersections_feed_the_device_batch_like_the_host_batch(k):
    """II_IntersectBatchDevice -> TopKFilteredBatchDevice equals II_IntersectBatch -> TopKFilteredBatch.  The result sets are
    released with FreeAfter right after the enqueue, before anything is synchronised."""
    import torch
    from redisearch_b200 import postings as ps

    vs = _vs()
    rng = np.random.default_rng(7)
    g, _ = _fp32_index()
    for lab in rng.choice(np.arange(1, 60_001), 500, replace=False).tolist():
        g.delete(int(lab))
    pool, pls = _pool_lists(rng, 60_000)
    nq = 40
    pairs = [(int(rng.integers(0, len(pool))), int(rng.integers(0, len(pool)))) for _ in range(nq)]
    pairs[0], pairs[1] = (0, 6), (4, 5)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, 64)
    # the host path
    P, L = ps.lib(), vs.lib()
    arrays = [(C.c_void_p * 2)(pls[a].h, pls[b].h) for a, b in pairs]
    lists_pp = (C.c_void_p * nq)(*[C.cast(a, C.c_void_p) for a in arrays])
    n_lists = (C.c_size_t * nq)(*([2] * nq))
    rs_out = (C.c_void_p * nq)()
    assert P.II_IntersectBatch(nq, lists_pp, n_lists, rs_out) == nq
    q_ptrs = (C.c_void_p * nq)(*[qs[i].ctypes.data for i in range(nq)])
    id_ptrs, counts = (C.c_void_p * nq)(), (C.c_size_t * nq)()
    for i in range(nq):
        counts[i] = P.II_ResultSet_Len(rs_out[i])
        id_ptrs[i] = P.II_ResultSet_DeviceDocIds(rs_out[i]) if counts[i] else None
    out_l = np.zeros((nq, k), dtype=np.uint64)
    out_s = np.zeros((nq, k), dtype=np.float64)
    out_c = (C.c_size_t * nq)()
    assert L.VecSimB200_TopKFilteredBatch(g.h, q_ptrs, nq, k, id_ptrs, counts, out_l.ctypes.data, out_s.ctypes.data, out_c) == 0
    for i in range(nq):
        P.II_ResultSet_Free(rs_out[i])
    # the device path, on a stream of its own
    s = torch.cuda.Stream()
    qd = _dev(stored_queries(g, qs))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        res = ps.intersect_batch_device([[pls[a], pls[b]] for a, b in pairs], stream=s)
        # an AND with the empty list (pool index 6) has no set: its cap is 0
        assert [r[0] is None for r in res] == [6 in p for p in pairs]
        labels, scores, dcounts, rc = g.topk_filtered_batch_device(qd, k, [r[1] for r in res], [r[3] for r in res],
                                                                   counts=[r[2] for r in res], stream=s)
        assert rc == 0
        for r in res:
            if r[0] is not None:
                r[0].free_after(s)
    s.synchronize()
    labels, scores, dcounts = labels.cpu().numpy(), scores.cpu().numpy(), dcounts.cpu().numpy()
    for i in range(nq):
        c = int(out_c[i])
        assert dcounts[i] == c, i
        assert labels[i, :c].tolist() == out_l[i, :c].astype(np.int64).tolist(), i
        assert scores[i, :c].tobytes() == out_s[i, :c].astype(np.float32).tobytes(), i
        assert (labels[i, c:] == -1).all() and np.isnan(scores[i, c:]).all(), i


def test_caps_above_the_counts_and_exact_caps_give_the_same_answers():
    rng = np.random.default_rng(9)
    g, _ = _fp32_index()
    filters = [np.sort(rng.choice(np.arange(1, 70_000), s, replace=False)).astype(np.uint32) for s in (0, 3, 50, 2000, 30_000)]
    qs = ol.synth_rows(ol.F32, 44, 0, len(filters), 64)
    for k in (10, 300):
        base = device_batch(g, qs, k, filters)
        big = device_batch(g, qs, k, filters, caps=[len(f) * 13 + 1000 for f in filters])
        exact = device_batch(g, qs, k, filters, exact_caps=True)
        for a, b in ((base, big), (base, exact)):
            assert a[0].tolist() == b[0].tolist() and a[1].tobytes() == b[1].tobytes() and a[2].tolist() == b[2].tolist()
        for i, f in enumerate(filters):
            assert_row_equals_filtered(g, qs[i], k, f, base[0][i], base[1][i], base[2][i], (k, i))


def test_neither_entry_point_waits_for_the_device():
    """With the index flushed and the scratch grown, both calls return while the caller's stream is still spinning."""
    import torch
    from redisearch_b200 import postings as ps

    rng = np.random.default_rng(11)
    g, _ = _fp32_index()
    pool, pls = _pool_lists(rng, 60_000)
    pairs = [(0, 1), (2, 1), (3, 0), (1, 2)]
    batch = [[pls[a], pls[b]] for a, b in pairs]
    nq, k = len(batch), 10
    qs = ol.synth_rows(ol.F32, 45, 0, nq, 64)
    qd = _dev(stored_queries(g, qs))
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    out_c = torch.empty(nq, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()

    def run():
        res = ps.intersect_batch_device(batch, stream=s)
        rc = g.topk_filtered_batch_device(qd, k, [r[1] for r in res], [r[3] for r in res], counts=[r[2] for r in res],
                                          out_labels=out_l, out_scores=out_s, out_counts=out_c, stream=s)[3]
        for r in res:
            r[0].free_after(s)
        return rc

    assert run() == 0  # warm-up: pools, scratch and staging at this size
    s.synchronize()
    want = (out_l.cpu().numpy().copy(), out_s.cpu().numpy().copy())
    out_l.fill_(7)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)  # ~0.1 s of spinning ahead of the batch
    assert run() == 0
    busy = not s.query()
    s.synchronize()
    assert busy, "an entry point waited for the caller's stream"
    assert out_l.cpu().numpy().tolist() == want[0].tolist() and out_s.cpu().numpy().tobytes() == want[1].tobytes()
    for i, (a, b) in enumerate(pairs):
        f = np.intersect1d(pool[a], pool[b]).astype(np.uint32)
        assert_row_equals_filtered(g, qs[i], k, f, want[0][i], want[1][i], int(out_c[i].item()), i)


@pytest.mark.parametrize("k", [10, 1000])
def test_launch_count_does_not_depend_on_the_batch_size(k):
    rng = np.random.default_rng(13)
    g, _ = _fp32_index()
    pool = [np.sort(rng.choice(np.arange(1, 60_001), s, replace=False)).astype(np.uint32) for s in (5000, 800, 20_000, 0)]
    launches = []
    for nq in (16, 256):
        filters = [pool[i % len(pool)] for i in range(nq)]
        qs = ol.synth_rows(ol.F32, 46, 0, nq, 64)
        device_batch(g, qs, k, filters)  # warm-up
        g.stats(reset=True)
        device_batch(g, qs, k, filters)
        launches.append(g.stats(reset=True).kernel_launches)
    assert launches[0] == launches[1] == 2 + 2 * ((k + 127) // 128), launches


def test_limits():
    import torch

    vs = _vs()
    g, _ = _fp32_index(n=2000)
    qd = _dev(stored_queries(g, ol.synth_rows(ol.F32, 47, 0, 2, 64)))
    f = _dev(np.arange(1, 101, dtype=np.int32))
    assert g.topk_filtered_batch_device(qd, 1025, [f.data_ptr()] * 2, [100, 100])[3] == -1
    torch.cuda.synchronize()
    g.stats(reset=True)
    assert g.topk_filtered_batch_device(qd, 10, [], [])[3] == 0  # nq = 0
    assert g.topk_filtered_batch_device(qd, 0, [f.data_ptr()] * 2, [100, 100])[3] == 0  # k = 0
    assert g.stats(reset=True).kernel_launches == 0
    assert g.topk_filtered_batch_device(qd, 10, [f.data_ptr()] * 2, [100, 2**32])[3] == -2  # a cap beyond the 32-bit ids
    sparse = vs.VecSimIndex(vs.VecSimType_FLOAT32, 64, vs.VecSimMetric_Cosine)
    rows = ol.synth_rows(ol.F32, 48, 0, 2, 64)
    assert sparse.add_many(rows, labels=np.array([1, 2**32 + 5], dtype=np.uint64)) == 2
    out_l = torch.full((2, 10), 7, dtype=torch.int64, device="cuda")
    rc = sparse.topk_filtered_batch_device(qd, 10, [f.data_ptr()] * 2, [100, 100], out_labels=out_l)[3]
    torch.cuda.synchronize()
    assert rc == -2 and (out_l == 7).all().item()  # refused before anything was enqueued
    assert sparse.stats(reset=True).kernel_launches == 0


@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
def test_mutations_between_batches_show_up_in_the_next_batch(multi):
    vs = _vs()
    rng = np.random.default_rng(17)
    dim, n = 32, 5000
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2, multi=multi)
    rows = ol.synth_rows(ol.F32, 49, 0, n, dim)
    assert g.add_many(rows, label0=1) == n
    qs = ol.synth_rows(ol.F32, 50, 0, 3, dim)
    filters = [np.arange(1, n + 20, dtype=np.uint32), np.arange(1, n + 20, 7, dtype=np.uint32), np.array([3, 4, 5], dtype=np.uint32)]

    def check(stage):
        for k in (10, 200):
            labels, scores, counts = device_batch(g, qs, k, filters)
            for i, f in enumerate(filters):
                assert_row_equals_filtered(g, qs[i], k, f, labels[i], scores[i], counts[i], (stage, k, i))

    check("fresh")
    near = qs[0] + np.float32(1e-3)
    assert g.add(near, n + 10) == 1  # a new docId, nearest to query 0
    check("add")
    labels, _, _ = device_batch(g, qs, 1, filters)
    assert labels[0, 0] == n + 10
    g.add(qs[2], 4)  # raw overwrite of docId 4 (single-value) / a second row for it (multi-value)
    check("overwrite")
    labels, scores, _ = device_batch(g, qs, 1, filters)
    assert labels[2, 0] == 4 and scores[2, 0] == 0.0
    for lab in set(rng.choice(np.arange(1, n), 300, replace=False).tolist()) | {4}:
        g.delete(int(lab))  # swap-delete moves the last rows into the holes
    check("delete")
    labels, _, _ = device_batch(g, qs, 1, filters)
    assert labels[2, 0] != 4


def test_accessors_on_pending_result_sets_match_the_host_batch():
    from redisearch_b200 import postings as ps

    rng = np.random.default_rng(19)
    pool, pls = _pool_lists(rng, 60_000)
    pairs = [(0, 1), (2, 3), (1, 4), (0, 6)]
    batch = [[pls[a], pls[b]] for a, b in pairs]
    P = ps.lib()
    nq = len(batch)
    arrays = [ps._list_array(b) for b in batch]
    lists_pp = (C.c_void_p * nq)(*[C.cast(a, C.c_void_p) for a in arrays])
    n_lists = (C.c_size_t * nq)(*[len(b) for b in batch])
    host = (C.c_void_p * nq)()
    assert P.II_IntersectBatch(nq, lists_pp, n_lists, host) == nq
    dev = ps.intersect_batch_device(batch)
    assert dev[3][0] is None and dev[3][3] == 0  # the empty list
    for i in range(3):
        rs = dev[i][0]
        assert dev[i][3] >= len(rs)
        assert len(rs) == P.II_ResultSet_Len(host[i]) == len(np.intersect1d(pool[pairs[i][0]], pool[pairs[i][1]]))
        ids, _, freqs = rs.fetch()
        h = ps.ResultSet(host[i])
        hids, _, hfreqs = h.fetch()
        assert ids.tolist() == hids.tolist() and freqs.tolist() == hfreqs.tolist()
        h.close()
        rs.close()
    P.II_ResultSet_Free(host[3])
    # a pending set read straight away, before any synchronisation
    rs = ps.intersect_batch_device([batch[0]])[0][0]
    assert rs.fetch(want_freqs=False)[0].tolist() == np.intersect1d(pool[0], pool[1]).tolist()
    rs.close()
