"""Batches of OR and numeric-range pre-filters on the device with no host wait: II_UnionBatchDevice and
II_NumericFilterBatchDevice, alone and feeding VecSimB200_TopKFilteredBatchDevice.

Every settled set must be the one II_Union builds (docIds, count, child freq rows, child order, num_estimated, scores), every
numeric set the one II_Union(quick) builds over II_NumericList_Filter of its leaves, and every KNN row the one
VecSimB200_TopKFiltered gives on the host-built filter, bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol

U32_MAX_ID = 2**32 - 2


# ------------------------------------------------------------------------------------------------
# CPU: the models the GPU tests lean on
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_oracle_union_is_the_set_union(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 30))
    lists = [np.unique(rng.integers(1, 5000, int(rng.integers(0, 400)))) for _ in range(n)]
    idx = [ol.InvIndex(ol.CODEC_FREQS_ONLY, l, np.ones(len(l), dtype=np.uint32)) for l in lists]
    want = np.unique(np.concatenate(lists)) if any(len(l) for l in lists) else np.zeros(0, dtype=np.int64)
    for quick in (False, True):
        got = ol.run_intersect(idx, union=True, quick=quick)
        assert [d for d, _ in got] == want.tolist()
        if not quick:
            for d, ch in got[:: max(1, len(got) // 50)]:
                assert sorted(c for c, _ in ch) == [j for j, l in enumerate(lists) if d in set(l.tolist())]


def in_range(values, lo, hi, lo_incl, hi_incl):
    """numpy model of NumericFilter::value_in_range"""
    v = np.asarray(values, dtype=np.float64)
    return ((v > lo) | (bool(lo_incl) & (v == lo))) & ((v < hi) | (bool(hi_incl) & (v == hi)))


def numeric_model(leaves, lo, hi, lo_incl, hi_incl):
    """ascending docIds with at least one value in range in any leaf; leaves = [(docIds, values)]"""
    hits = [ids[in_range(vals, lo, hi, lo_incl, hi_incl)] for ids, vals in leaves]
    return np.unique(np.concatenate(hits)).astype(np.uint64) if hits else np.zeros(0, dtype=np.uint64)


def test_numeric_model_agrees_with_the_oracle_range_test():
    rng = np.random.default_rng(3)
    P = ol.postings()
    vals = np.concatenate([rng.normal(0, 100, 300), [np.inf, -np.inf, 0.0, -0.0, 5.0, 5.0, 1e300, -1e300]])
    bounds = [(-10.0, 10.0), (5.0, 5.0), (10.0, -10.0), (-np.inf, np.inf), (np.inf, np.inf), (-np.inf, -np.inf), (0.0, 0.0), (-0.0, 0.0)]
    for lo, hi in bounds:
        for li in (0, 1):
            for hi_ in (0, 1):
                want = [bool(P.orc_numeric_in_range(float(v), lo, hi, li, hi_)) for v in vals]
                assert in_range(vals, lo, hi, li, hi_).tolist() == want, (lo, hi, li, hi_)
    # multi-value documents: one hit per document, whatever the number of its values in range
    ids = np.array([1, 1, 1, 4, 4, 9], dtype=np.uint64)
    v = np.array([1.0, 2.0, 50.0, np.inf, 3.0, -np.inf])
    assert numeric_model([(ids, v), (ids[:3], v[:3])], 0, 10, 1, 1).tolist() == [1, 4]
    assert numeric_model([(ids, v)], -np.inf, np.inf, 1, 1).tolist() == [1, 4, 9]
    assert numeric_model([(ids, v)], -np.inf, np.inf, 0, 0).tolist() == [1, 4]
    assert numeric_model([(ids, v)], 10, 0, 1, 1).tolist() == []


# ------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------
def _ps():
    from redisearch_b200 import postings as ps

    return ps


def _writer_list(ids, freqs):
    ps = _ps()
    w = ps.IndexWriter(ps.CODEC_FREQS_ONLY)
    for d, f in zip(ids.tolist(), freqs.tolist()):
        w.add(int(d), int(f))
    return ps.PostingList.from_blocks(w.blocks(), ps.CODEC_FREQS_ONLY, on_device=True)


_POOL = {}


def zipf_pool(universe=12_000, n=400):
    """n posting lists from the index writer with Zipf sizes (universe / 2, / 4, ...) over docIds 1..universe"""
    key = (universe, n)
    if key not in _POOL:
        rng = np.random.default_rng(universe + n)
        arrays, lists = [], []
        for i in range(n):
            size = max(1, int(universe / 2 / (i + 1) ** 1.1))
            ids = np.unique(rng.integers(1, universe + 1, size)).astype(np.uint64)
            freqs = rng.integers(1, 20, len(ids)).astype(np.uint32)
            arrays.append((ids, freqs))
            lists.append(_writer_list(ids, freqs))
        _POOL[key] = (arrays, lists)
    return _POOL[key]


def _host_union(lists, quick):
    ps = _ps()
    return ps.ResultSet(ps.lib().II_Union(ps._list_array(lists), len(lists), int(quick)))


def _num_estimated(rs, n_children):
    """num_estimated of a full-mode set, through the list view II_ResultSet_IntoChild makes of it (consumes rs)"""
    pl = rs.into_child([(1.0, 1.0, 1.0)] * n_children)
    return pl.num_estimated(), pl


def assert_same_set(dev, host, quick, freqs=True, what=None):
    assert len(dev) == len(host), what
    ids, _, fr = dev.fetch(want_freqs=not quick and freqs)
    hids, _, hfr = host.fetch(want_freqs=not quick and freqs)
    assert ids.tolist() == hids.tolist(), what
    if not quick and freqs:
        assert fr.tobytes() == hfr.tobytes(), what
    assert dev.child_order().tolist() == host.child_order().tolist(), what
    L = _ps().lib()
    assert L.II_ResultSet_Capacity(dev.h) == L.II_ResultSet_Capacity(host.h), what
    return ids


def _spin(stream, cycles=200_000_000):
    import torch

    with torch.cuda.stream(stream):
        torch.cuda._sleep(cycles)  # ~0.1 s of spinning ahead of the batch


# ------------------------------------------------------------------------------------------------
# GPU: union parity
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("quick", [False, True], ids=["full", "quick"])
@pytest.mark.parametrize("n_lists", [1, 2, 20, 21, 200, 1024])
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_union_batch_equals_ii_union(nq, n_lists, quick):
    """Every set equals II_Union on the same lists.  Freq rows are compared whole where a set has at most 2^20 entries, and
    on every 16th query of the wide 256-query batches (their scores cover every row, test_union_batch_scores_like_ii_union)."""
    arrays, pool = zipf_pool()
    rng = np.random.default_rng(nq * 10_000 + n_lists * 2 + quick)
    picks = [rng.choice(len(pool), n_lists, replace=n_lists > len(pool)).tolist() for _ in range(nq)]
    batch = [[pool[j] for j in p] for p in picks]
    res = _ps().union_batch_device(batch, quick_exit=quick)
    for i, (rs, d_ids, d_len, cap) in enumerate(res):
        assert rs is not None and d_ids and d_len and cap > 0
        host = _host_union(batch[i], quick)
        want = np.unique(np.concatenate([arrays[j][0] for j in picks[i]]))
        full_rows = n_lists * len(want) <= 1 << 20 or i % 16 == 0
        ids = assert_same_set(rs, host, quick, freqs=full_rows, what=(i, n_lists))
        assert ids.tolist() == want.tolist()
        if not quick and n_lists <= 200 and i % 8 == 0:
            ne, _ = _num_estimated(rs, n_lists)
            assert ne == _num_estimated(host, n_lists)[0] == sum(len(arrays[j][0]) for j in picks[i])


@pytest.mark.gpu
@pytest.mark.parametrize("n_lists", [2, 20, 21, 200])
def test_union_batch_scores_like_ii_union(n_lists):
    """II_Score over the batch's sets: BM25STD, TFIDF and DISMAX bits equal II_Union's (the per-child freqs, the child order of
    every docId epoch and the wide-union tables all enter the scores)."""
    ps = _ps()
    arrays, pool = zipf_pool()
    rng = np.random.default_rng(50 + n_lists)
    nq, n_docs = 16, 12_000
    picks = [rng.choice(len(pool), n_lists, replace=False).tolist() for _ in range(nq)]
    batch = [[pool[j] for j in p] for p in picks]
    doc_len = rng.integers(1, 900, n_docs + 1).astype(np.uint32)
    dt = ps.DocTable(n_docs, doc_len, rng.choice(np.array([1.0, 0.5, 0.1], dtype=np.float32), n_docs + 1),
                     rng.integers(1, 60, n_docs + 1).astype(np.uint32))
    P = ol.postings()
    for scorer in (ps.SCORER_BM25STD, ps.SCORER_TFIDF, ps.SCORER_DISMAX):
        res = ps.union_batch_device(batch)
        for i, p in enumerate(picks):
            terms = [(float(rng.choice([1.0, 0.5, 2.0])), P.orc_idf(n_docs, len(arrays[j][0])), P.orc_idf_bm25(n_docs, len(arrays[j][0])))
                     for j in p]
            host = _host_union(batch[i], False)
            rs = res[i][0]
            for s in (rs, host):
                s.score(scorer, terms, 0.7, n_docs, 123.25, dt)
            a, b = rs.fetch(want_freqs=False), host.fetch(want_freqs=False)
            assert a[0].tolist() == b[0].tolist() and a[1].tobytes() == b[1].tobytes(), (scorer, i)


@pytest.mark.gpu
def test_union_batch_into_child_scores_like_ii_union():
    """IntoChild of a full-mode set inside an II_Intersect scores like the one made from II_Union"""
    ps = _ps()
    arrays, pool = zipf_pool()
    rng = np.random.default_rng(77)
    n_docs = 12_000
    picks = [[0, 3, 9], [1, 2, 5, 8, 13, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57]]
    other = _writer_list(np.arange(1, n_docs + 1, 2, dtype=np.uint64), rng.integers(1, 9, n_docs // 2).astype(np.uint32))
    res = ps.union_batch_device([[pool[j] for j in p] for p in picks])
    doc_len = rng.integers(1, 900, n_docs + 1).astype(np.uint32)
    dt = ps.DocTable(n_docs, doc_len)
    P = ol.postings()
    for i, p in enumerate(picks):
        inner_terms = [(1.0, P.orc_idf(n_docs, len(arrays[j][0])), P.orc_idf_bm25(n_docs, len(arrays[j][0]))) for j in p]
        outer_terms = [(1.0, 0.0, 0.0), (1.0, P.orc_idf(n_docs, len(other)), P.orc_idf_bm25(n_docs, len(other)))]
        got = []
        for rs in (res[i][0], _host_union([pool[j] for j in p], False)):
            child = rs.into_child(inner_terms, 0.5)
            assert child.num_estimated() == sum(len(arrays[j][0]) for j in p)
            top = ps.intersect([child, other])
            top.score(ps.SCORER_BM25STD, outer_terms, 1.0, n_docs, 200.0, dt)
            got.append(top.fetch())
        assert got[0][0].tolist() == got[1][0].tolist() and got[0][1].tobytes() == got[1][1].tobytes()
        assert got[0][2].tobytes() == got[1][2].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("quick", [False, True], ids=["full", "quick"])
def test_union_batch_edge_inputs(quick):
    ps = _ps()
    _, pool = zipf_pool()
    empty = ps.PostingList.from_arrays([], [])
    lo = ps.PostingList.from_arrays([1, 2, 5], [3, 1, 2])
    hi = ps.PostingList.from_arrays([7, U32_MAX_ID], [4, 9])
    shared = pool[1]
    batch = [
        [empty],                      # all lists empty: no set
        [empty, empty, empty],
        [],                           # no list
        [pool[3], empty, pool[3]],    # the same list twice, an empty one between
        [lo, hi],                     # docIds 1 and 2^32 - 2 in one window
        [hi],
        [empty, lo],
    ] + [[shared, pool[10 + i]] for i in range(12)]  # one list shared by every query
    res = ps.union_batch_device(batch, quick_exit=quick)
    for i, lists in enumerate(batch):
        rs, _, _, cap = res[i]
        if not lists or all(len(l) == 0 for l in lists):
            assert rs is None and cap == 0, i
            continue
        assert_same_set(rs, _host_union(lists, quick), quick, what=i)
    assert res[4][0].fetch(want_freqs=False)[0].tolist() == [1, 2, 5, 7, U32_MAX_ID]


# ------------------------------------------------------------------------------------------------
# GPU: numeric parity
# ------------------------------------------------------------------------------------------------
def price_leaves(rng, n_docs=20_000, n_leaves=24):
    """A synthetic multi-value price field split into leaves by value, as a range tree splits it: a document with several prices
    sits in several leaves (or repeats inside one); +-inf prices included.  Returns [(docIds, values)], [NumericList]."""
    ps = _ps()
    per_doc = rng.integers(1, 4, n_docs)
    docs = np.repeat(np.arange(1, n_docs + 1, dtype=np.uint64), per_doc)
    prices = np.round(rng.lognormal(4, 1, len(docs)), 2)
    prices[rng.choice(len(prices), 40, replace=False)] = np.inf
    prices[rng.choice(len(prices), 40, replace=False)] = -np.inf
    edges = np.quantile(prices[np.isfinite(prices)], np.linspace(0, 1, n_leaves + 1))[1:-1]
    leaf_of = np.searchsorted(edges, prices)
    arrays, leaves = [], []
    for L in range(n_leaves):
        sel = leaf_of == L
        ids, vals = docs[sel], prices[sel]
        order = np.argsort(ids, kind="stable")
        ids, vals = ids[order], vals[order]
        w = ps.IndexWriter(numeric=True)
        for d, v in zip(ids.tolist(), vals.tolist()):
            w.add_numeric(int(d), v)
        arrays.append((ids, vals))
        leaves.append(ps.NumericList(w.blocks()))
    return arrays, leaves, prices


def numeric_queries(rng, prices, n_leaves, nq):
    """(leaf indices, lo, hi, lo_incl, hi_incl): ranges of 0 %, 1 % and 100 %, bounds on present values, +-inf, min > max"""
    finite = np.sort(prices[np.isfinite(prices)])
    out = []
    for i in range(nq):
        kind = i % 6
        if kind == 0:    # ~1 % of the values, inclusive, bounds on present values
            a = int(rng.integers(0, len(finite) - len(finite) // 100))
            q = (finite[a], finite[a + len(finite) // 100], 1, 1)
        elif kind == 1:  # the same, exclusive
            a = int(rng.integers(0, len(finite) - len(finite) // 100))
            q = (finite[a], finite[a + len(finite) // 100], 0, 0)
        elif kind == 2:  # 100 %
            q = (-np.inf, np.inf, 1, 1)
        elif kind == 3:  # 0 %: min > max
            q = (500.0, 10.0, 1, 1)
        elif kind == 4:  # 0 %: a gap between values
            q = (1e12, 2e12, 1, 1)
        else:            # everything above a price, +inf included
            q = (finite[len(finite) // 2], np.inf, 0, 1)
        picks = sorted(rng.choice(n_leaves, int(rng.integers(1, n_leaves + 1)), replace=False).tolist())
        out.append((picks,) + q)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_numeric_filter_batch_equals_union_of_filtered_leaves(nq):
    ps = _ps()
    rng = np.random.default_rng(nq)
    arrays, leaves, prices = price_leaves(rng)
    qs = numeric_queries(rng, prices, len(leaves), nq)
    res = ps.numeric_filter_batch_device([([leaves[j] for j in p], lo, hi, li, hi_) for p, lo, hi, li, hi_ in qs])
    for i, (p, lo, hi, li, hi_) in enumerate(qs):
        want = numeric_model([arrays[j] for j in p], lo, hi, li, hi_)
        filtered = [leaves[j].filter(lo, hi, li, hi_) for j in p]
        host = _host_union(filtered, True)
        rs, _, _, cap = res[i]
        assert rs is not None and cap >= len(want)
        assert len(rs) == len(host) == len(want), (i, lo, hi, li, hi_)
        ids = rs.fetch(want_freqs=False)[0]
        assert ids.tolist() == host.fetch(want_freqs=False)[0].tolist() == want.tolist(), i
        assert rs.child_order().tolist() == list(range(len(p)))


# ------------------------------------------------------------------------------------------------
# GPU: end to end, and no host wait
# ------------------------------------------------------------------------------------------------
def _index(kind, n=60_000, dim=64):
    from redisearch_b200 import vecsim as vs

    if kind == "f32_cos":
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
        assert g.add_many(rows, label0=1) == n
        return g, ol.synth_rows(ol.F32, 43, 0, 64, dim)
    if kind == "i8_l2":
        g = vs.VecSimIndex(vs.VecSimType_INT8, dim, vs.VecSimMetric_L2)
        rows = ol.synth_rows(ol.I8, 42, 0, n, dim)
        assert g.add_many(rows, label0=1) == n
        return g, ol.synth_rows(ol.I8, 43, 0, 64, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2, multi=True)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    labels = (np.arange(n, dtype=np.uint64) // 3 + 1)[np.random.default_rng(5).permutation(n)]
    assert g.add_many(rows, labels=labels) == n
    return g, ol.synth_rows(ol.F32, 43, 0, 64, dim)


_LEAVES = {}


def cached_leaves(n_docs, n_leaves, seed=7):
    key = (n_docs, n_leaves, seed)
    if key not in _LEAVES:
        _LEAVES[key] = price_leaves(np.random.default_rng(seed), n_docs=n_docs, n_leaves=n_leaves)
    return _LEAVES[key]


def _filter_batch(rng, n_docs, stream=None):
    """12 tag-style ORs over a Zipf pool of docIds up to n_docs and 12 price ranges over leaves of the same documents, as
    pending sets whose events `stream` waits for; and the filters they must hold"""
    ps = _ps()
    u_arrays, u_pool = zipf_pool(universe=n_docs, n=120)
    n_arrays, leaves, prices = cached_leaves(n_docs, 12)
    ors = [rng.choice(len(u_pool), int(rng.integers(1, 40)), replace=False).tolist() for _ in range(12)]
    ranges = numeric_queries(rng, prices, len(leaves), 12)
    sets = ps.union_batch_device([[u_pool[j] for j in p] for p in ors], quick_exit=True, stream=stream)
    sets += ps.numeric_filter_batch_device([([leaves[j] for j in p], lo, hi, li, hi_) for p, lo, hi, li, hi_ in ranges], stream=stream)
    want = [np.unique(np.concatenate([u_arrays[j][0] for j in p])).astype(np.uint32) for p in ors]
    want += [numeric_model([n_arrays[j] for j in p], lo, hi, li, hi_).astype(np.uint32) for p, lo, hi, li, hi_ in ranges]
    return sets, want


def _knn_on_sets(g, qd, k, sets, stream, **outs):
    """TopKFilteredBatchDevice over the sets' device docIds / counts / caps, then FreeAfter on every set at once"""
    labels, scores, counts, rc = g.topk_filtered_batch_device(qd, k, [r[1] for r in sets], [r[3] for r in sets],
                                                              counts=[r[2] for r in sets], stream=stream, **outs)
    for r in sets:
        if r[0] is not None:
            r[0].free_after(stream)
    return labels, scores, counts, rc


@pytest.mark.gpu
@pytest.mark.parametrize("k", [10, 1000])
@pytest.mark.parametrize("kind", ["f32_cos", "i8_l2", "f32_multi"])
def test_device_filters_feed_the_device_knn_like_the_host_filters(kind, k):
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries

    g, qs_all = _index(kind)
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    sets, want = _filter_batch(np.random.default_rng(len(kind) + k), 70_000, stream=s)
    labels, scores, counts, rc = _knn_on_sets(g, qd, k, sets, s)
    assert rc == 0
    s.synchronize()
    labels, scores, counts = labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], k, f, labels[i], scores[i], int(counts[i]), (kind, k, i))


@pytest.mark.gpu
def test_no_entry_point_waits_for_the_callers_stream():
    """With a kernel still spinning on the caller's stream, both filter calls and the KNN return before it ends; the answers
    are right afterwards."""
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries

    g, qs_all = _index("f32_cos")
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    outs = dict(out_labels=torch.empty((24, 10), dtype=torch.int64, device="cuda"),
                out_scores=torch.empty((24, 10), dtype=torch.float32, device="cuda"),
                out_counts=torch.empty(24, dtype=torch.int32, device="cuda"))
    s = torch.cuda.Stream()
    sets, _ = _filter_batch(np.random.default_rng(21), 70_000, stream=s)  # warm-up: pools, scratch and staging at this size
    assert _knn_on_sets(g, qd, 10, sets, s, **outs)[3] == 0
    s.synchronize()
    outs["out_labels"].fill_(7)
    torch.cuda.synchronize()
    _spin(s)
    sets, want = _filter_batch(np.random.default_rng(21), 70_000, stream=s)
    rc = _knn_on_sets(g, qd, 10, sets, s, **outs)[3]
    busy = not s.query()
    s.synchronize()
    assert rc == 0
    assert busy, "an entry point waited for the caller's stream"
    labels, scores, counts = (outs[n].cpu().numpy() for n in ("out_labels", "out_scores", "out_counts"))
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], 10, f, labels[i], scores[i], int(counts[i]), i)


@pytest.mark.gpu
def test_launches_do_not_depend_on_the_batch_size_or_the_lists():
    ps = _ps()
    _, pool = zipf_pool()
    rng = np.random.default_rng(31)
    arrays, leaves, prices = price_leaves(rng, n_docs=5000, n_leaves=8)
    for quick, per_batch in ((False, 6), (True, 4)):
        seen = []
        for nq in (16, 256):
            for n_lists in (2, 200):
                batch = [[pool[j] for j in rng.choice(len(pool), n_lists, replace=False).tolist()] for _ in range(nq)]
                ps.stats(reset=True)
                res = ps.union_batch_device(batch, quick_exit=quick)
                seen.append(ps.stats(reset=True).kernel_launches)
                assert all(r[0] is not None for r in res)
                del res
        assert seen == [per_batch] * 4, (quick, seen)
    seen = []
    for nq in (16, 256):
        qs = numeric_queries(rng, prices, len(leaves), nq)
        ps.stats(reset=True)
        ps.numeric_filter_batch_device([([leaves[j] for j in p], lo, hi, li, hi_) for p, lo, hi, li, hi_ in qs])
        seen.append(ps.stats(reset=True).kernel_launches)
    assert seen == [4, 4]


@pytest.mark.gpu
def test_argument_errors_are_refused_before_any_launch():
    ps = _ps()
    _, pool = zipf_pool()
    L = ps.lib()
    too_many = [pool[i % len(pool)] for i in range(1025)]
    nested = ps.union([pool[0], pool[1]]).into_child([(1.0, 1.0, 1.0)] * 2)
    for batch in ([[pool[0]], too_many], [[pool[2], nested]]):
        ps.stats(reset=True)
        with pytest.raises(ValueError):
            ps.union_batch_device(batch)
        assert ps.stats(reset=True).kernel_launches == 0
    # a NULL leaf / no ranges
    out = (C.c_void_p * 1)()
    leaf_pp = (C.c_void_p * 1)(None)
    tab = (C.c_void_p * 1)(C.cast(leaf_pp, C.c_void_p))
    n = (C.c_size_t * 1)(1)
    rng = (ps.II_NumericRange * 1)(ps.II_NumericRange(0.0, 1.0, 1, 1))
    assert L.II_NumericFilterBatchDevice(1, tab, n, rng, None, out, None) == -1
    assert L.II_UnionBatchDevice(0, None, None, 0, None, out, None) == 0
    assert ps.stats(reset=True).kernel_launches == 0
