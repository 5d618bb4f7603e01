"""Hybrid KNN batches on two device routes (VecSimB200_HybridTopKBatchDevice, DESIGN.md §4.10).

Each query takes the ragged gather of VecSimB200_TopKFilteredBatchDevice or the filtered tensor-core route (row-space filter
bitmaps, filtered sample pass, fixed-bound main pass with the filter bit on its survivor path, exact rescoring selected by
(distance, docId), the second tier, and the gather for what stays open).  Every answer row must equal, bit for bit, the row
VecSimB200_TopKFilteredBatchDevice returns for the same query and filter: labels, distance bits, counts.

The CPU tests model the filtered sample -> bound -> keep -> proof chain in numpy, with ties and random filter fractions, and the
host's sample sizing and cap floor.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from test_hybrid_device_batch import _dev, device_batch, stored_queries
from test_vecsim_large_k_batch import clustered_corpus

QN = 128          # rows per row tile (coarse_tc.cu kQN)
EPS_F16 = 1.2e-3  # |approx - exact| bound of the fp16 route for unit rows (coarse_tc.h kCoarseEpsF16)
SLICES = 32       # slice minima per (query, row range) of the sample pass
EMPTY_MODE, HYBRID_ADHOC_BF, HYBRID_BATCHES = 0, 2, 3


# ------------------------------------------------------------------------------------------------------------------
# CPU model (vecsim_index.cpp hybrid_topk_batch_device / sample_stride; coarse_tc.cu kFilt)
# ------------------------------------------------------------------------------------------------------------------
def tiles_per_k(k):
    return 1 / 32.0 if k > 128 else 2.0


def cap_floor(k):
    return int(np.ceil(tiles_per_k(k) * k * QN / 0.25))


def sample_stride(tiles, ranges, k, aim, tpk):
    f = min(0.25, max(0.01, k / (aim * ranges)))
    return int(max(1.0, min(np.floor(1 / f), np.floor(tiles / (tpk * k)))))


def filtered_chain(approx, exact, filt, k, ranges, eps):
    """One query of the dense route with k <= 128: the filtered sample pass (slice minima over filtered rows only), the bound,
    the main pass's keep set, the refine's (distance, docId) selection and its proof.  filt: bool per row.  Returns
    (proven, answer rows) with answer = the k smallest (exact, docId) among the kept rows; docId = row here."""
    n = approx.shape[0]
    tiles = (n + QN - 1) // QN
    f = max(filt.mean(), 1e-9)
    stride = sample_stride(tiles, ranges, k, 24.0, tiles_per_k(k) / f)
    tile_of = np.arange(n) // QN
    sampled = (tile_of % stride == 0) & filt
    visit = tile_of // stride  # the sample's own tile counter
    slice_id = (visit % ranges) * SLICES + ((visit // ranges) % 8) * 4 + (np.arange(n) % QN) // 32
    minima = {}
    for r in np.nonzero(sampled)[0]:
        s = slice_id[r]
        minima[s] = min(minima.get(s, np.inf), approx[r])
    m = np.sort(np.array(list(minima.values()), dtype=np.float64))
    T = m[k - 1] + 2 * eps if m.size >= k else np.inf
    kept = np.nonzero(filt & (approx < T))[0]
    order = np.lexsort((kept, exact[kept]))
    ans = kept[order][:k]
    proven = np.isfinite(T) and ans.size >= k and T - eps > exact[ans[-1]]
    return proven, ans


@pytest.mark.parametrize("seed", range(6))
def test_filtered_bound_keeps_every_row_of_the_gathers_answer(seed):
    """With approximations within eps of the exact distances, a proven query's kept rows hold the gather's whole answer: every
    filtered row at or below the k-th filtered exact distance, exact ties included, so (distance, docId) over the kept rows equals
    (distance, position) over the ascending filter."""
    rng = np.random.default_rng(seed)
    n, ranges = 200_000, 33
    exact = rng.random(n).astype(np.float64)
    # ties: a block of identical distances straddling the k-th place of the filter
    tie_rows = rng.choice(n, 400, replace=False)
    frac = [0.002, 0.01, 0.1, 0.5, 1.0][seed % 5]
    filt = rng.random(n) < frac
    k = int(rng.choice([1, 10, 128]))
    fe = np.sort(exact[filt])
    exact[tie_rows] = fe[min(k, fe.size) - 1] if fe.size else 0.5
    eps = EPS_F16
    approx = exact + rng.uniform(-eps, eps, n)
    proven, ans = filtered_chain(approx, exact, filt, k, ranges, eps)
    frows = np.nonzero(filt)[0]  # ascending docIds = ascending positions
    g = frows[np.lexsort((np.arange(frows.size), exact[frows]))][:k]
    if proven:
        assert ans.tolist() == g.tolist()
        ek = exact[g[-1]]
        assert np.all(np.isin(frows[exact[frows] <= ek], ans) | (exact[frows[exact[frows] <= ek]] == ek))
    assert proven or frac < 0.01 or filt.sum() < k


def test_sample_sizing_and_cap_floor():
    """At the cap floor the stride stays >= 4 (the sample is at most a quarter of the corpus) and the sample visits
    tiles_per_k / f times the tiles of the unfiltered route: about 256 k filtered rows for k <= 128, 4 k for k > 128."""
    for n in (70_000, 300_000, 10_000_000):
        tiles = (n + QN - 1) // QN
        for k in (1, 10, 128, 129, 1000, 1024):
            cap = cap_floor(k)
            if cap > n:
                continue
            f = cap / n
            aim = 128.0 if k > 128 else 24.0
            s = sample_stride(tiles, 33, k, aim, tiles_per_k(k) / f)
            assert s >= 4 or tiles / (tiles_per_k(k) / f * k) < 4.0 + 1e-9, (n, k, s)
            filtered_in_sample = tiles / s * QN * f
            assert filtered_in_sample >= (4 * k if k > 128 else 2 * k), (n, k, s, filtered_in_sample)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


@pytest.fixture
def mode1():
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    yield vs
    vs.lib().VecSimB200_SetCoarseMode(-1)


def _params(policy):
    vs = _vs()
    if policy is None:
        return None
    p = vs.VecSimQueryParams()
    p.searchMode = policy
    return p


def hybrid_batch(g, qs, k, filters, policy=None, caps=None, exact_caps=False, stream=None):
    """One VecSimB200_HybridTopKBatchDevice call (device_batch's arguments); returns labels, scores, counts, modes, flags."""
    import torch

    bufs, cnts, ptrs, cps, cptrs = [], [], [], [], []
    for i, f in enumerate(filters):
        cap = len(f) if caps is None else caps[i]
        buf = np.full(max(cap, 1), 0xFFFFFFF0, dtype=np.uint32)
        buf[: len(f)] = f
        bufs.append(_dev(buf.view(np.int32)))
        cnts.append(_dev(np.array([len(f)], dtype=np.int32)))
        ptrs.append(bufs[-1].data_ptr() if cap else None)
        cptrs.append(cnts[-1].data_ptr())
        cps.append(cap)
    qd = _dev(stored_queries(g, qs))
    labels, scores, counts, modes, rc = g.hybrid_topk_batch_device(qd, k, ptrs, cps, counts=None if exact_caps else cptrs,
                                                                   params=_params(policy), stream=stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    flags = np.zeros(len(filters), dtype=np.uint32)
    assert g.L.VecSimB200_LastCoarseFlags(g.h, flags.ctypes.data_as(C.c_void_p), len(filters)) == 0
    return labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy().astype(np.int64), modes, flags


def assert_equal_rows(g, qs, k, filters, policy=None, caps=None, exact_caps=False):
    """Hybrid rows == TopKFilteredBatchDevice rows: labels, score bits, counts.  Returns (modes, flags)."""
    want = device_batch(g, qs, k, filters, caps=caps, exact_caps=exact_caps)
    got = hybrid_batch(g, qs, k, filters, policy=policy, caps=caps, exact_caps=exact_caps)
    assert got[0].tolist() == want[0].tolist()
    assert got[1].tobytes() == want[1].tobytes()
    assert got[2].tolist() == want[2].tolist()
    return got[3], got[4]


def _index(metric, n, dim, vtype=ol.F32, multi=False, seed=42, deletes=True):
    """docIds 1..n; with `deletes`, 200 swap-deletes (the last rows move into the holes) so labels no longer follow rows."""
    vs = _vs()
    g = vs.VecSimIndex(vtype, dim, metric, multi=multi)
    rows = ol.synth_rows(vtype, seed, 0, n, dim)
    if multi:
        assert g.add_many(rows, labels=(np.arange(n, dtype=np.uint64) // 2 + 1)) == n
    else:
        assert g.add_many(rows, label0=1) == n
    deleted = []
    if deletes and not multi:
        deleted = list(range(1, n, n // 200))[:200]
        for d in deleted:
            assert g.delete(d) == 1
    return g, set(deleted)


def _filters(rng, top, nq, k, fracs):
    """Ascending filters over docIds 1..top + 100 (the tail is absent), cycling through the fractions; 'lt_k' = fewer than k."""
    out = []
    for i in range(nq):
        fr = fracs[i % len(fracs)]
        if fr == "empty":
            out.append(np.zeros(0, np.uint32))
        elif fr == "lt_k":
            out.append(np.sort(rng.choice(np.arange(1, top + 101), max(0, k - 1), replace=False)).astype(np.uint32))
        else:
            m = min(top + 100, max(1, int(fr * top)))
            out.append(np.sort(rng.choice(np.arange(1, top + 101), m, replace=False)).astype(np.uint32))
    return out


FRACS = ["empty", "lt_k", 0.001, 0.01, 0.1, 0.5, 1.0]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["cosine", "ip", "l2"])
@pytest.mark.parametrize("k", [1, 10, 128, 129, 1000, 1024])
def test_forced_dense_rows_equal_the_gather(mode1, metric, k):
    vs = mode1
    m = {"cosine": vs.VecSimMetric_Cosine, "ip": vs.VecSimMetric_IP, "l2": vs.VecSimMetric_L2}[metric]
    rng = np.random.default_rng(k)
    g, _ = _index(m, 70_000, 128)
    nq = 40
    qs = ol.synth_rows(ol.F32, 7, 0, nq, 128)
    filters = _filters(rng, 70_000, nq, k, FRACS)
    modes, flags = assert_equal_rows(g, qs, k, filters, policy=HYBRID_BATCHES)
    assert (modes == HYBRID_BATCHES).all()
    assert g.L.VecSimB200_LastBatchPath(g.h) == 1
    big = [i for i, f in enumerate(filters) if len(f) >= 7000]
    assert all(flags[i] in (1, 2) for i in big), flags  # broad filters are proven on the tensor cores
    for policy in (None, HYBRID_ADHOC_BF):
        assert_equal_rows(g, qs, k, filters, policy=policy)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [32, 768, 1016])
@pytest.mark.parametrize("k", [10, 1000])
def test_dims(mode1, dim, k):
    vs = mode1
    rng = np.random.default_rng(dim)
    g, _ = _index(vs.VecSimMetric_Cosine, 70_000, dim)
    qs = ol.synth_rows(ol.F32, 8, 0, 16, dim)
    filters = _filters(rng, 70_000, 16, k, [0.01, 0.1, 0.5, 1.0])
    modes, flags = assert_equal_rows(g, qs, k, filters, policy=HYBRID_BATCHES)
    assert (modes == HYBRID_BATCHES).all() and (flags > 0).sum() >= 8, flags


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [16, 256])
@pytest.mark.parametrize("k", [10, 1000])
def test_large_corpus_automatic_plan(mode1, nq, k):
    """300K rows: the automatic plan sends broad filters to the dense route and narrow ones to the gather, and the rows match."""
    vs = mode1
    rng = np.random.default_rng(nq + k)
    g, _ = _index(vs.VecSimMetric_Cosine, 300_000, 128)
    qs = ol.synth_rows(ol.F32, 9, 0, nq, 128)
    filters = _filters(rng, 300_000, nq, k, [0.001, 0.5])
    broad = [i for i, f in enumerate(filters) if len(f) > 100_000]
    modes, flags = assert_equal_rows(g, qs, k, filters)
    if len(broad) < 16:  # too few dense queries to pay for the first shadow build: all on the gather
        assert (modes == HYBRID_ADHOC_BF).all(), modes
        qd = _dev(stored_queries(g, qs[:1].repeat(16, axis=0)))
        import torch

        lab = torch.empty((16, k), dtype=torch.int64, device="cuda")
        scr = torch.empty((16, k), dtype=torch.float32, device="cuda")
        assert g.L.VecSimB200_TopKQueryBatchDevice(g.h, C.c_void_p(qd.data_ptr()), 16, k, C.c_void_p(lab.data_ptr()),
                                                   C.c_void_p(scr.data_ptr()), None) == 0  # builds the shadow
        modes, flags = assert_equal_rows(g, qs, k, filters)
    floor = cap_floor(k)
    for i, f in enumerate(filters):
        if len(f) < floor:
            assert modes[i] == HYBRID_ADHOC_BF and flags[i] == 0
    assert (modes[broad] == HYBRID_BATCHES).all() and (flags[broad] > 0).all(), (modes, flags)


@pytest.mark.gpu
def test_ties_resolve_by_docid(mode1):
    """Duplicate rows whose labels were permuted against the rows by swap-deletes, straddling the k-th place."""
    vs = mode1
    dim, n = 64, 70_000
    rows = ol.synth_rows(ol.F32, 3, 0, n, dim)
    dup = rows[5].copy()
    rng = np.random.default_rng(5)
    pos = rng.choice(np.arange(100, n), 60, replace=False)
    rows[pos] = dup
    g = vs.VecSimIndex(ol.F32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == n
    for d in rng.choice(np.arange(1, n + 1), 300, replace=False):
        g.delete(int(d))
    q = dup + np.float32(1e-3) * ol.synth_rows(ol.F32, 4, 0, 1, dim)[0]
    qs = np.repeat(q[None, :], 16, axis=0)
    filters = [np.arange(1, n + 1, dtype=np.uint32)[rng.random(n) < 0.6] for _ in range(16)]
    for k in (10, 30, 129):
        modes, flags = assert_equal_rows(g, qs, k, filters, policy=HYBRID_BATCHES)
        assert (flags > 0).any()


@pytest.mark.gpu
def test_overflow_goes_to_the_second_tier_and_the_gather(mode1):
    """clustered_corpus with every docId in the filter: qa's tied block defeats both tiers (flag 0, the gather answers), qb's
    block overflows the main pass and the second tier proves it (flag 2)."""
    vs = mode1
    rows, qa, qb = clustered_corpus(300_000, 128)
    g = vs.VecSimIndex(ol.F32, 128, vs.VecSimMetric_Cosine)
    n = rows.shape[0]
    assert g.add_many(rows, label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, 40, 128)
    qs[:8] = qa
    qs[8:16] = qb
    filt = np.arange(1, n + 1, dtype=np.uint32)
    modes, flags = assert_equal_rows(g, qs, 256, [filt] * 40, policy=HYBRID_BATCHES)
    assert (flags[:8] == 0).all() and (flags[8:16] == 2).all(), flags.tolist()


@pytest.mark.gpu
def test_caps_and_counts(mode1):
    """Caps far above the counts, a small filter forced dense through an inflated cap, and no count pointers."""
    vs = mode1
    rng = np.random.default_rng(21)
    g, _ = _index(vs.VecSimMetric_L2, 70_000, 64)
    qs = ol.synth_rows(ol.F32, 13, 0, 16, 64)
    filters = _filters(rng, 70_000, 16, 10, [0.001, 0.3])
    caps = [len(f) * 4 + 60_000 for f in filters]
    modes, _ = assert_equal_rows(g, qs, 10, filters, caps=caps)
    assert (modes == HYBRID_BATCHES).all()
    assert_equal_rows(g, qs, 10, filters, exact_caps=True)
    assert_equal_rows(g, qs, 10, filters, exact_caps=True, policy=HYBRID_BATCHES)


@pytest.mark.gpu
def test_policies_and_rule_boundary(mode1):
    """The automatic plan follows the cap floor on both sides of it; the three policies give the same rows."""
    vs = mode1
    rng = np.random.default_rng(22)
    n = 300_000
    g, _ = _index(vs.VecSimMetric_Cosine, n, 128)
    qs = ol.synth_rows(ol.F32, 14, 0, 32, 128)
    fl = cap_floor(10)
    sizes = [fl - 1] * 16 + [150_000] * 16
    filters = [np.sort(rng.choice(np.arange(1, n + 1), s, replace=False)).astype(np.uint32) for s in sizes]
    modes, _ = assert_equal_rows(g, qs, 10, filters)
    assert (modes[:16] == HYBRID_ADHOC_BF).all() and (modes[16:] == HYBRID_BATCHES).all(), modes
    for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
        m2, f2 = assert_equal_rows(g, qs, 10, filters, policy=policy)
        assert (m2 == policy).all()
        if policy == HYBRID_ADHOC_BF:
            assert (f2 == 0).all() and g.L.VecSimB200_LastBatchPath(g.h) == 0
    p = _params(5)
    lab, sc, cn, md, rc = g.hybrid_topk_batch_device(_dev(stored_queries(g, qs[:1])), 10, [0], [0], params=p)
    assert rc == -1


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fp16", "int8", "multi", "mode0", "mode2", "small", "subset", "range"])
def test_ineligible_batches_take_the_gather(case):
    vs = _vs()
    rng = np.random.default_rng(23)
    mode = {"mode0": 0, "mode2": 2}.get(case, 1)
    vs.lib().VecSimB200_SetCoarseMode(mode)
    try:
        vtype = {"fp16": ol.F16, "int8": ol.I8}.get(case, ol.F32)
        metric = vs.VecSimMetric_L2 if case in ("int8", "range") else vs.VecSimMetric_IP
        n = 60_000 if case == "small" else 70_000
        g, _ = _index(metric, n, 64, vtype=vtype, multi=case == "multi", deletes=False)
        if case == "range":  # a row beyond the fp16 range
            big = np.full((1, 64), 70_000.0, dtype=np.float32)
            assert g.add_many(big, label0=n + 1) == 1
        nq = 8 if case == "subset" else 16
        qs = ol.synth_rows(vtype, 15, 0, nq, 64)
        top = n // 2 if case == "multi" else n
        filters = _filters(rng, top, nq, 10, [0.5])
        modes, flags = assert_equal_rows(g, qs, 10, filters, policy=HYBRID_BATCHES)
        assert (modes == HYBRID_ADHOC_BF).all() and (flags == 0).all(), case
        assert g.L.VecSimB200_LastBatchPath(g.h) == 0
    finally:
        vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
def test_pending_filters_from_the_posting_lists(mode1):
    """AND, OR and filter-mode AND results of the device posting-list batches feed the call while still pending."""
    import torch
    from redisearch_b200 import postings as ps

    vs = mode1
    rng = np.random.default_rng(24)
    n = 70_000
    g, _ = _index(vs.VecSimMetric_Cosine, n, 64, deletes=False)
    pool = [np.sort(rng.choice(np.arange(1, n + 1), s, replace=False)).astype(np.uint64) for s in (60_000, 50_000, 40_000)]
    pls = [ps.PostingList.from_arrays(p) for p in pool]
    batch = [[pls[i % 3], pls[(i + 1) % 3]] for i in range(16)]
    qs = ol.synth_rows(ol.F32, 16, 0, 16, 64)
    qd = _dev(stored_queries(g, qs))
    for kind in ("and", "or"):
        res = ps.intersect_batch_device(batch) if kind == "and" else ps.union_batch_device(batch)
        lab, sc, cn, md, rc = g.hybrid_topk_batch_device(qd, 10, [r[1] for r in res], [r[3] for r in res], counts=[r[2] for r in res],
                                                         params=_params(HYBRID_BATCHES))
        assert rc == 0
        torch.cuda.synchronize()
        fn = np.intersect1d if kind == "and" else np.union1d
        filters = [fn(pool[i % 3], pool[(i + 1) % 3]).astype(np.uint32) for i in range(16)]
        want = device_batch(g, qs, 10, filters)
        for r in res:
            r[0].free_after(None)
        assert lab.cpu().numpy().tolist() == want[0].tolist() and sc.cpu().numpy().tobytes() == want[1].tobytes(), kind
        assert (md == HYBRID_BATCHES).all()


@pytest.mark.gpu
def test_no_host_wait_and_launches_independent_of_nq(mode1):
    import torch

    vs = mode1
    rng = np.random.default_rng(25)
    n = 70_000
    g, _ = _index(vs.VecSimMetric_Cosine, n, 64)
    launches = []
    for nq in (16, 256):
        qs = ol.synth_rows(ol.F32, 17, 0, nq, 64)
        filters = _filters(rng, n, nq, 10, [0.01, 0.5])
        hybrid_batch(g, qs, 10, filters, policy=HYBRID_BATCHES)  # warm-up
        g.stats(reset=True)
        hybrid_batch(g, qs, 10, filters, policy=HYBRID_BATCHES)
        launches.append(g.stats(reset=True).kernel_launches)
    assert launches[0] == launches[1] == 14 + 2, launches
    # no host wait: the call returns while the caller's stream spins
    nq, k = 16, 10
    qs = ol.synth_rows(ol.F32, 18, 0, nq, 64)
    filters = _filters(rng, n, nq, k, [0.5])
    bufs = [_dev(f.view(np.int32)) for f in filters]
    qd = _dev(stored_queries(g, qs))
    s = torch.cuda.Stream()
    out = [torch.empty((nq, k), dtype=torch.int64, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
           torch.empty(nq, dtype=torch.int32, device="cuda")]

    def run():
        return g.hybrid_topk_batch_device(qd, k, [b.data_ptr() for b in bufs], [len(f) for f in filters], params=_params(HYBRID_BATCHES),
                                          out_labels=out[0], out_scores=out[1], out_counts=out[2], stream=s)[4]

    assert run() == 0
    s.synchronize()
    want = out[0].cpu().numpy().copy()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
    assert run() == 0
    busy = not s.query()
    s.synchronize()
    assert busy, "the call waited for the caller's stream"
    assert out[0].cpu().numpy().tolist() == want.tolist()


@pytest.mark.gpu
def test_mutations_and_shared_scratch(mode1):
    """Appends, an overwrite and a swap-delete between batches; interleaved with the other device batch calls on one stream."""
    import torch

    vs = mode1
    rng = np.random.default_rng(26)
    n, dim = 70_000, 64
    g, _ = _index(vs.VecSimMetric_Cosine, n, dim)
    qs = ol.synth_rows(ol.F32, 19, 0, 16, dim)
    filters = _filters(rng, n + 2000, 16, 10, [0.5, 1.0])
    assert_equal_rows(g, qs, 10, filters, policy=HYBRID_BATCHES)
    assert g.add_many(ol.synth_rows(ol.F32, 20, 0, 2000, dim), label0=n + 1) == 2000
    g.add(qs[0], 7)  # overwrite: docId 7 is now the first query itself
    g.delete(int(filters[1][3]))
    modes, flags = assert_equal_rows(g, qs, 10, filters, policy=HYBRID_BATCHES)
    assert (flags > 0).any()
    qd = _dev(stored_queries(g, qs))
    lab = torch.empty((16, 10), dtype=torch.int64, device="cuda")
    scr = torch.empty((16, 10), dtype=torch.float32, device="cuda")
    assert g.L.VecSimB200_TopKQueryBatchDevice(g.h, C.c_void_p(qd.data_ptr()), 16, 10, C.c_void_p(lab.data_ptr()),
                                               C.c_void_p(scr.data_ptr()), None) == 0
    assert_equal_rows(g, qs, 10, filters, policy=HYBRID_BATCHES)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_against_the_reference(mode1):
    """8 queries: ids and score bits against the reference's distance over the rows read back from the device, in (distance,
    docId) order."""
    vs = mode1
    rng = np.random.default_rng(27)
    n, dim = 70_000, 128
    g, _ = _index(vs.VecSimMetric_L2, n, dim, deletes=False)
    qs = ol.synth_rows(ol.F32, 28, 0, 16, dim)
    filters = _filters(rng, n, 16, 10, [0.02, 0.3])
    lab, sc, cn, modes, flags = hybrid_batch(g, qs, 10, filters, policy=HYBRID_BATCHES)
    assert (flags > 0).sum() >= 8
    o = ol.RefIndex(ol.F32, dim, ol.L2) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, dim, ol.L2, tier=ol.TIER_AVX512)
    rows = np.empty((n, dim), dtype=np.float32)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, rows.ctypes.data_as(C.c_void_p)) == 0
    o.add_many(rows, 1)  # no deletes: row r holds docId r + 1
    for i in range(8):
        f = filters[i]
        d = np.array([np.float32(o.distance_from(int(x), qs[i])) for x in f.tolist()], dtype=np.float32)
        order = np.lexsort((f, d))[:10]
        assert lab[i].tolist() == f[order].astype(np.int64).tolist(), i
        assert sc[i].tobytes() == d[order].tobytes(), i
