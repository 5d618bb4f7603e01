"""KNN batches with 128 < k <= 1024 on the device (DESIGN.md §4.5).

Single-value fp32 batches the fp32 route serves (coarse mode 1, fixed bound, nq >= 16, >= 65,536 rows, dim % 8 == 0, 32..1024)
take the two-pass route with lists of 256 per (query, row range) and the wide refine; the queries it leaves open finish on the
batched exact top-k (one score scan per group of queries + ceil(k / 128) cursor selects), on the device.  The device API answers
every other single-value batch with that exact top-k.  Every answer must equal, in ids and float32 score bits, the per-query
VecSimIndex_TopKQuery(k) on the same index and the reference's scan (oracle/_ref when built, else the C restatement at the
AVX-512 tier) over the rows read back from the device.
"""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as ol

SIZE_MAX = np.uint64(0xFFFFFFFFFFFFFFFF)
QN = 128            # rows per row tile of the main pass (coarse_tc.cu kQN)
LIST_CAP = 256      # list slots per (query, row range) of the main pass for k > 128
EPS_F16 = 1.2e-3    # |approx - exact| bound of the fp16 route for unit rows (coarse_tc.h kCoarseEpsF16)
H100_SMS = 132
_METRICS = {"cosine": ol.COS, "ip": ol.IP, "l2": ol.L2}
_KEEPALIVE = []  # timeout callbacks stay registered with the library after a test ends


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


@pytest.fixture
def mode1():
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    yield vs
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# helpers (CPU)
# ------------------------------------------------------------------------------------------------------------------
def select_k(labels, scores, k):
    """The k best (score, label) pairs, ascending by score then label: the reference's order."""
    labels, scores = np.asarray(labels, dtype=np.int64), np.asarray(scores, dtype=np.float32)
    order = np.lexsort((labels, scores))[:k]
    return labels[order], scores[order]


def _unit(x):
    x = np.asarray(x, dtype=np.float64)
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def clustered_corpus(n, dim, seed=0):
    """Random rows, then two contiguous blocks of 40,000 rows each (the row ranges of the main pass visit interleaved tiles, so a
    contiguous block puts ~300 rows into every range):
      block A  copies of one row at cosine distance 0.3 from query qa: their exact ties fill every list of both tiers below the
               k-th distance, so neither proof holds and the query takes the exact fallback (flag 0);
      block B  distinct rows at distances 0.78 .. 0.79 from query qb, beyond its k-th distance among the random rows (~0.73 at dim
               128) but below the main pass's bound: every list of the main pass overflows, and the second tier's lists of 128
               end well beyond the k-th distance, so the second tier proves the query (flag 2).
    Returns (rows fp32 [n + 80000][dim], qa, qb)."""
    rng = np.random.default_rng(seed)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim).astype(np.float32)
    qa, qb = _unit(rng.standard_normal(dim)), _unit(rng.standard_normal(dim))

    def at_distance(q, d, u):
        u = u - np.outer(u @ q, q)
        u = _unit(u)
        c = 1.0 - d
        return (c[:, None] * q[None, :] + np.sqrt(1.0 - c * c)[:, None] * u).astype(np.float32)

    m = 40_000
    a = at_distance(qa, np.array([0.3]), rng.standard_normal((1, dim)))
    block_a = np.repeat(a, m, axis=0)
    block_b = at_distance(qb, np.linspace(0.78, 0.79, m), rng.standard_normal((m, dim)))
    return np.concatenate([rows, block_a, block_b]), qa.astype(np.float32), qb.astype(np.float32)


def simulate_main_pass(dist, k, ranges, eps=EPS_F16):
    """Per-(query, row range) count of rows the main pass keeps (approx < T), with the plan of batch_scan_rows for k > 128 and the
    exact distances standing in for the fp16 ones: sample = adaptive lists of 128 per range over every stride-th tile, T = the
    k-th smallest of their union + 2 eps.  dist: one query's distances over the corpus in row order."""
    n = dist.shape[0]
    tiles = (n + QN - 1) // QN
    f = min(0.25, max(0.01, k / (128.0 * ranges)))
    stride = int(max(1, min(np.floor(1 / f), np.floor(tiles / (k / 32.0)))))
    tile_of = np.arange(n) // QN
    sampled = tile_of % stride == 0
    s_tiles = (tiles + stride - 1) // stride
    s_ranges = min(s_tiles, ranges)
    s_range = (tile_of // stride) % s_ranges
    union = []
    for r in range(s_ranges):
        d = dist[sampled & (s_range == r)]
        union.append(np.sort(d)[:128])
    union = np.sort(np.concatenate(union))
    T = union[k - 1] + 2 * eps if union.size >= k else np.inf
    kept = dist < T
    return np.bincount((tile_of % ranges)[kept], minlength=ranges)


# ------------------------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "ip", "l2"])
@pytest.mark.parametrize("k", [129, 300, 1000, 1024])
def test_selection_helper_equals_the_reference(metric, k):
    dim, n = 32, 1500
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    rows[700:760] = rows[100:160]  # exact ties: the lower label first
    ref = ol.RefIndex(ol.F32, dim, _METRICS[metric]) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, dim, _METRICS[metric])
    port = ol.PortIndex(ol.F32, dim, _METRICS[metric])
    ref.add_many(rows, 1)
    port.add_many(rows, 1)
    for qi, q in enumerate(ol.synth_rows(ol.F32, 43, 0, 4, dim)):
        if qi == 1:
            q = rows[120].copy()
        al, as_ = port.all_sorted(q)
        hl, hs = select_k(al, as_.astype(np.float32), k)
        rl, rs = ref.topk(q, k)
        assert hl.tolist() == rl.astype(np.int64).tolist()
        assert hs.tobytes() == rs.astype(np.float32).tobytes()


def test_clustered_builder_overflows_the_main_pass():
    """Block A and B queries keep more than 256 rows in a row range of the main pass (the fallback and the second tier are
    exercised); random queries stay within the lists."""
    n, dim, k = 300_000, 128, 256
    rows, qa, qb = clustered_corpus(n, dim)
    u = _unit(rows)
    ranges = H100_SMS  # nq <= 64: one query group, one row range per SM
    for q, overflow in ((qa, True), (qb, True), (_unit(ol.synth_rows(ol.F32, 43, 0, 1, dim)[0]), False)):
        dist = (1.0 - u @ _unit(q)).astype(np.float32)
        cnt = simulate_main_pass(dist, k, ranges)
        assert (cnt.max() > LIST_CAP) == overflow, (overflow, int(cnt.max()))
    # block B lies beyond the k-th distance of its query: the second tier's lists end beyond it
    dist_b = (1.0 - u @ _unit(qb)).astype(np.float32)
    assert np.sort(dist_b[:n])[k - 1] + 2 * EPS_F16 < 0.78


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _index(metric, dim, rows):
    vs = _vs()
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, {"cosine": vs.VecSimMetric_Cosine, "ip": vs.VecSimMetric_IP, "l2": vs.VecSimMetric_L2}[metric])
    assert g.add_many(rows, label0=1) == len(rows)
    return g


def _read_rows(g, n, dim):
    out = np.empty((n, dim), dtype=np.float32)
    assert _vs().lib().VecSimB200_ReadRows(g.h, 0, n, out.ctypes.data) == 0
    return out


def _stored_queries(metric, qs):
    qs = np.array(qs, dtype=np.float32, copy=True)
    if metric == "cosine":
        for i in range(len(qs)):
            ol.port().orc_normalize(ol._p(qs[i]), qs.shape[1], ol.F32)
    return qs


def _reference(metric, g, n, dim, qs, k):
    """The reference's scan over the device's stored rows: [(labels, scores)] per query."""
    s = ol.StreamingTopK(ol.F32, _METRICS[metric], dim, _stored_queries(metric, qs), k, os.cpu_count() or 1)
    s.feed(_read_rows(g, n, dim), 1)
    return [s.result(i) for i in range(len(qs))]


def _device_batch(g, qs_stored, k):
    import torch

    vs = _vs()
    nq = qs_stored.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qs_stored).view(np.uint8).copy()).cuda()  # stored-form rows, pitch 16-aligned here
    out_l = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    out_s = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp)
    torch.cuda.synchronize()
    if rc != 0:
        return rc, None, None, None
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(g.h, flags.ctypes.data, nq)
    return 0, out_l.cpu().numpy(), out_s.cpu().numpy(), (flags if frc == 0 else None)


def _path(g):
    return _vs().lib().VecSimB200_LastBatchPath(g.h)


def _same(hl, hs, dl, ds):
    """host API ([nq][k] uint64 / float64, SIZE_MAX / NaN padded) == device API (int64 / float32, -1 / NaN padded)"""
    h = hl != SIZE_MAX
    assert ((dl >= 0) == h).all()
    assert (dl[h].astype(np.uint64) == hl[h]).all() and ds[h].tobytes() == hs[h].astype(np.float32).tobytes()


def _check_row(labels, scores, want_l, want_s, tag):
    h = labels != SIZE_MAX if labels.dtype == np.uint64 else labels >= 0
    gl, gs = labels[h].astype(np.int64), scores[h].astype(np.float32)
    assert gl.tolist() == np.asarray(want_l, dtype=np.int64).tolist(), (tag, gl[:6].tolist(), list(want_l[:6]))
    assert gs.tobytes() == np.asarray(want_s, dtype=np.float32).tobytes(), tag


def _per_query(g, qs, k):
    out = []
    for q in qs:
        ids, scores, code = g.topk(q, k)
        assert code == 0
        out.append((ids.astype(np.int64), scores.astype(np.float32)))
    return out


# ------------------------------------------------------------------------------------------------------------------
# GPU: parity matrix
# ------------------------------------------------------------------------------------------------------------------
_BATCHES = [(16, 129), (40, 256), (256, 1000), (256, 1024), (16, 1024), (40, 1000), (256, 129), (40, 129), (16, 256), (256, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["cosine", "ip", "l2"])
@pytest.mark.parametrize("dim", [32, 128, 768, 1016])
@pytest.mark.parametrize("n", [70_000, 300_000])
def test_matrix_is_exact(mode1, metric, dim, n):
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    rows[5000:5040] = rows[4000:4040]  # exact duplicates: the lower id wins
    g = _index(metric, dim, rows)
    qs_all = ol.synth_rows(ol.F32, 43, 0, 256, dim)
    qs_all[1] = rows[4003]
    ref = _reference(metric, g, n, dim, qs_all, 1024)
    one = _per_query(g, qs_all, 1024)  # VecSimIndex_TopKQuery(1024); its first k are TopKQuery(k) (same total order)
    for i in (0, 1, 255):
        l, s = g.topk(qs_all[i], 300)[:2]
        assert l.astype(np.int64).tolist() == one[i][0][:300].tolist() and s.astype(np.float32).tobytes() == one[i][1][:300].tobytes()
    for nq, k in _BATCHES:
        qs = np.ascontiguousarray(qs_all[:nq])
        hl, hs, rc = g.topk_batch(qs, k)
        assert rc == 0 and _path(g) == 1, (nq, k)
        rc, dl, ds, flags = _device_batch(g, _stored_queries(metric, qs), k)
        assert rc == 0 and _path(g) == 1 and flags is not None, (nq, k)
        assert (flags != 0).sum() >= 0.9 * nq, (nq, k, np.bincount(flags, minlength=3).tolist())
        _same(hl, hs, dl, ds)
        for i in range(nq):
            _check_row(hl[i], hs[i], one[i][0][:k], one[i][1][:k], ("per-query", nq, k, i))
            _check_row(hl[i], hs[i], ref[i][0][:k], ref[i][1][:k], ("reference", nq, k, i))


# ------------------------------------------------------------------------------------------------------------------
# GPU: ties, clustered corpora, the fp16 range
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_duplicates_straddle_the_kth_boundary(mode1):
    n, dim, nq, k = 300_000, 128, 32, 1000
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    u = _unit(rows)
    d0 = 1.0 - u @ _unit(qs[0])
    r = int(np.argsort(d0, kind="stable")[990])  # a row near query 0's k-th place
    spots = np.random.default_rng(3).choice(n, 60, replace=False)
    rows[spots] = rows[r]  # 61 copies spread over the row ranges: ranks ~990 .. ~1050 tie
    g = _index("cosine", dim, rows)
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 1
    tied = np.sort(np.concatenate([spots, [r]])) + 1
    row0 = hl[0].astype(np.int64)
    inside = np.isin(tied, row0)
    assert 0 < inside.sum() < len(tied)  # the boundary cuts the copies ...
    assert inside[: inside.sum()].all()  # ... and keeps the lowest labels
    one = _per_query(g, qs, k)
    ref = _reference("cosine", g, n, dim, qs, k)
    for i in range(nq):
        _check_row(hl[i], hs[i], *one[i], ("per-query", i))
        _check_row(hl[i], hs[i], *ref[i], ("reference", i))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [256, 1000])
def test_clustered_corpus_reaches_tier2_and_the_fallback(mode1, k):
    n, dim, nq = 300_000, 128, 40
    rows, qa, qb = clustered_corpus(n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[:8] = qa
    qs[8:16] = qb
    g = _index("cosine", dim, rows)
    rc, dl, ds, flags = _device_batch(g, _stored_queries("cosine", qs), k)
    assert rc == 0 and _path(g) == 1 and flags is not None
    assert (flags[:8] == 0).all() and (flags[8:16] == 2).all(), flags.tolist()
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 1
    _same(hl, hs, dl, ds)
    one = _per_query(g, qs, k)
    ref = _reference("cosine", g, len(rows), dim, qs, k)
    for i in range(nq):
        _check_row(hl[i], hs[i], *one[i], ("per-query", i))
        _check_row(hl[i], hs[i], *ref[i], ("reference", i))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_queries_beyond_the_fp16_range_take_the_exact_path(mode1, metric):
    n, dim, nq, k = 70_000, 64, 32, 300
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[3, 5] = 65520.0
    qs[7, 0] = -70000.0
    g = _index(metric, dim, rows)
    rc, dl, ds, flags = _device_batch(g, qs, k)
    assert rc == 0 and _path(g) == 1 and flags is not None
    assert flags[3] == 0 and flags[7] == 0 and (np.delete(flags, [3, 7]) != 0).sum() >= 0.9 * (nq - 2), flags.tolist()
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0
    _same(hl, hs, dl, ds)
    one = _per_query(g, qs, k)
    ref = _reference(metric, g, n, dim, qs, k)
    for i in range(nq):
        _check_row(hl[i], hs[i], *one[i], ("per-query", i))
        _check_row(hl[i], hs[i], *ref[i], ("reference", i))


# ------------------------------------------------------------------------------------------------------------------
# GPU: the device API off the route, limits
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fp16", "int8", "mode0", "nq15", "rows500"])
def test_device_api_off_the_route_is_exact(mode1, case):
    vs = mode1
    dim, nq, k = 128, (15 if case == "nq15" else 32), (1000 if case == "rows500" else 300)
    n = 500 if case == "rows500" else 70_000
    vtype = {"fp16": ol.F16, "int8": ol.I8}.get(case, ol.F32)
    vst = {ol.F16: vs.VecSimType_FLOAT16, ol.I8: 4, ol.F32: vs.VecSimType_FLOAT32}[vtype]
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    g = vs.VecSimIndex(vst, dim, vs.VecSimMetric_IP)
    assert g.add_many(rows, label0=1) == n
    if case == "mode0":
        vs.lib().VecSimB200_SetCoarseMode(0)
    rc, dl, ds, flags = _device_batch(g, qs, k)
    assert rc == 0 and _path(g) == 0
    s = ol.StreamingTopK(vtype, ol.IP, dim, qs, k, os.cpu_count() or 1)
    stored = np.empty_like(rows)
    assert vs.lib().VecSimB200_ReadRows(g.h, 0, n, stored.ctypes.data) == 0
    s.feed(stored, 1)
    for i in range(nq):
        ids, scores, code = g.topk(qs[i], k)
        assert code == 0
        want = min(k, n)
        assert (dl[i, want:] == -1).all() and np.isnan(ds[i, want:]).all()  # fewer rows than k: the tail is padded
        _check_row(dl[i, :want], ds[i, :want], ids.astype(np.int64), scores.astype(np.float32), ("per-query", i))
        if vtype != ol.F16:  # fp16 scores are held to the project's 1e-2 bar against the reference, not to its bits
            _check_row(dl[i, :want], ds[i, :want], *s.result(i), ("reference", i))


@pytest.mark.gpu
def test_device_api_limits(mode1):
    vs = mode1
    dim, n = 64, 70_000
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = _stored_queries("cosine", ol.synth_rows(ol.F32, 43, 0, 16, dim))
    g = _index("cosine", dim, rows)
    assert _device_batch(g, qs, 1024)[0] == 0
    assert _device_batch(g, qs, 1025)[0] == -1
    m = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
    assert m.add_many(rows, labels=np.arange(n, dtype=np.uint64) // 2 + 1) == n
    assert _device_batch(m, qs, 128)[0] == 0
    assert _device_batch(m, qs, 129)[0] == -1


# ------------------------------------------------------------------------------------------------------------------
# GPU: mutations, timeouts, shards
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mutations_between_batches(mode1):
    """Appends, a raw overwrite of a resident row and a swap-delete between two k = 500 batches: the second equals the reference
    index that took the same mutations, and the per-query calls."""
    dim, n, nq, k = 128, 70_000, 32, 500
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    g = _index("l2", dim, rows)
    # the reference's own index when oracle/_ref is built (it takes the same adds, overwrites and deletes), else the C restatement
    p = ol.RefIndex(ol.F32, dim, ol.L2) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, dim, ol.L2)
    p.add_many(rows, 1)

    def batch(tag):
        hl, hs, rc = g.topk_batch(qs, k)
        assert rc == 0 and _path(g) == 1, tag
        rc, dl, ds, _ = _device_batch(g, qs, k)
        assert rc == 0, tag
        _same(hl, hs, dl, ds)
        for i in (0, 1, 2, 3, nq - 1):
            pl, ps = p.topk(qs[i], k)
            _check_row(hl[i], hs[i], pl, ps, (tag, i))
        return hl

    batch("fresh")
    more = ol.synth_rows(ol.F32, 44, 0, 2000, dim)
    more[7] = qs[0]
    for x in (g, p):
        x.add_many(more, label0=n + 1)  # appends, one a copy of query 0
        x.add(qs[1], 777)               # raw overwrite of a resident row
        x.delete(1000)                  # swap-delete: the last row moves into the hole
    hl = batch("mutated")
    assert hl[0, 0] == n + 8 and hl[1, 0] == 777 and not (hl == 1000).any()


@pytest.mark.gpu
def test_timeout_while_the_fallback_runs(mode1):
    vs = mode1
    L = vs.lib()
    n, dim, nq, k = 300_000, 128, 40, 1000
    rows, qa, qb = clustered_corpus(n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[:8] = qa  # these queries run the exact fallback
    g = _index("cosine", dim, rows)
    calls = {"n": 0}

    def fire_late(ctx):  # the first poll is the entry check; later ones come while the kernels run
        calls["n"] += 1
        return 1 if calls["n"] >= 2 else 0

    cb, cb_off = vs.TIMEOUT_CB(fire_late), vs.TIMEOUT_CB(lambda ctx: 0)
    _KEEPALIVE.extend([cb, cb_off])
    L.VecSim_SetTimeoutCallbackFunction(cb)
    try:
        qp = vs.VecSimQueryParams()
        _, _, rc = g.topk_batch(qs, k, C.byref(qp))
        assert rc == vs.VecSim_QueryReply_TimedOut and calls["n"] >= 2
    finally:
        L.VecSim_SetTimeoutCallbackFunction(cb_off)
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 1
    for i in (0, 8, nq - 1):
        ids, scores, code = g.topk(qs[i], k)
        _check_row(hl[i], hs[i], ids.astype(np.int64), scores.astype(np.float32), i)


@pytest.mark.gpu
def test_shard_groups_equal_the_single_index(mode1):
    import torch

    vs = mode1
    L = vs.lib()
    n, dim, nq, k = 140_000, 64, 32, 1000
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    one = _index("cosine", dim, rows)
    el, es, rc = one.topk_batch(qs, k)
    assert rc == 0 and _path(one) == 1
    grp = L.VecSimB200_ShardGroup_New(None, 0, 1)
    assert grp
    gl = np.zeros((nq, k), dtype=np.uint64)
    gs = np.zeros((nq, k), dtype=np.float64)
    assert L.VecSimB200_ShardGroup_TopKBatch(grp, one.h, qs.ctypes.data, qs.strides[0], nq, k, gl.ctypes.data, gs.ctypes.data) == 0
    L.VecSimB200_ShardGroup_Free(grp)
    assert (gl == el).all() and gs.astype(np.float32).tobytes() == es.astype(np.float32).tobytes()
    # two row shards on one GPU (labels kept), each answered on the device, merged as the shard group merges the exchange blocks
    block = int(L.VecSimB200_ShardBlockBytes(nq, k))
    buf = torch.zeros(2 * block, dtype=torch.uint8, device="cuda")
    qd = torch.from_numpy(_stored_queries("cosine", qs)).cuda()
    shards = []
    for s in range(2):
        ix = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        assert ix.add_many(rows[s::2], labels=np.arange(1 + s, n + 1, 2, dtype=np.uint64)) == n // 2
        shards.append(ix)
        lab = buf[s * block:s * block + nq * k * 8].view(torch.int64)
        sco = buf[s * block + nq * k * 8:s * block + nq * k * 12].view(torch.float32)
        sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert L.VecSimB200_TopKQueryBatchDevice(ix.h, qd.data_ptr(), nq, k, lab.data_ptr(), sco.data_ptr(), sp) == 0
        assert _path(ix) == 1
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.VecSimB200_MergeShardBlocks(buf.data_ptr(), 2, nq, k, out_s.data_ptr(), out_l.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    assert (out_l.cpu().numpy().astype(np.uint64) == el).all()
    assert out_s.cpu().numpy().tobytes() == es.astype(np.float32).tobytes()


_FIRST_WIDE_BATCH = r"""
import sys, os, ctypes as C
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch, oracle_lib as ol
from redisearch_b200 import vecsim as vs
L = vs.lib()
L.VecSimB200_SetCoarseMode(1)
n, dim, nq, k = 70_000, 128, 512, 300
rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, METRIC_VS)
assert g.add_many(rows, label0=1) == n
if API == "host":
    labels, scores, rc = g.topk_batch(qs, k)
    assert rc == 0, rc
else:
    qn = qs.copy()
    if METRIC_OL == ol.COS:
        for i in range(nq):
            ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    qd = torch.from_numpy(qn).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = L.VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp)
    torch.cuda.synchronize()
    assert rc == 0, rc
    labels, scores = out_l.cpu().numpy().astype(np.uint64), out_s.cpu().numpy()
assert L.VecSimB200_LastBatchPath(g.h) == 1
for i in (0, 1, 255, 256, 511):
    ids, sc, code = g.topk(qs[i], k)
    assert code == 0 and labels[i].astype(np.int64).tolist() == ids.tolist(), i
    assert scores[i].astype(np.float32).tobytes() == sc.astype(np.float32).tobytes(), i
print("FIRST-WIDE-OK")
"""


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("api", ["host", "device"])
def test_large_batch_is_the_first_wide_batch_of_its_process(metric, api):
    """512 queries: 8 query groups leave 16 row ranges, so the wide refine packs 4,096 candidates (32 KB) next to its 32 KB survivor
    buffer, above the 48 KB a launch gets without opting in.  Run as the first wide batch of a fresh process: no earlier launch
    has raised the kernel's limit."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    mvs = {"cosine": "vs.VecSimMetric_Cosine", "l2": "vs.VecSimMetric_L2"}[metric]
    mol = {"cosine": "ol.COS", "l2": "ol.L2"}[metric]
    head = f"ROOT = {root!r}\nAPI = {api!r}\n"
    code = _FIRST_WIDE_BATCH.replace("METRIC_VS", mvs).replace("METRIC_OL", mol)
    r = subprocess.run([sys.executable, "-c", head + code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "FIRST-WIDE-OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_device_api_batch_beyond_65535_queries(mode1):
    """A small corpus and 70,000 queries: every position in one group would put 70,000 slots on the chunk select's gridDim.y (limit
    65,535); groups are capped at 65,535 positions, so the batch runs as two groups."""
    import torch

    vs = mode1
    n, dim, nq, k = 500, 32, 70_000, 200
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2)
    assert g.add_many(rows, label0=1) == n
    qd = torch.from_numpy(qs).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    dl, ds = out_l.cpu().numpy(), out_s.cpu().numpy()
    for i in (0, 1, 65_534, 65_535, 65_536, nq - 1):
        ids, scores, code = g.topk(qs[i], k)
        assert code == 0
        _check_row(dl[i], ds[i], ids.astype(np.int64), scores.astype(np.float32), i)


_NCCL_WIDE = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol
from redisearch_b200 import vecsim as vs, sharding
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("gloo")
L = vs.lib()
L.VecSimB200_SetCoarseMode(1)
idbuf = np.zeros(128, dtype=np.uint8)
if rank == 0:
    assert L.VecSimB200_ShardGroup_UniqueId(idbuf.ctypes.data) == 0
t = torch.from_numpy(idbuf); dist.broadcast(t, 0)
g = L.VecSimB200_ShardGroup_New(idbuf.ctypes.data, rank, world)
assert g, "ncclCommInitRank failed"
N, DIM, K, B = 200_000, 64, 1000, 32
lo, hi = sharding.shard_range(N, world, rank)
qs = ol.synth_rows(ol.F32, 43, 0, B, DIM)
ix = vs.VecSimIndex(vs.VecSimType_FLOAT32, DIM, vs.VecSimMetric_Cosine)
ix.add_many(ol.synth_rows(ol.F32, 42, lo, hi - lo, DIM), label0=lo + 1)
labels = np.zeros((B, K), dtype=np.uint64); scores = np.zeros((B, K), dtype=np.float64)
assert L.VecSimB200_ShardGroup_TopKBatch(g, ix.h, qs.ctypes.data, qs.strides[0], B, K, labels.ctypes.data, scores.ctypes.data) == 0
one = vs.VecSimIndex(vs.VecSimType_FLOAT32, DIM, vs.VecSimMetric_Cosine)
one.add_many(ol.synth_rows(ol.F32, 42, 0, N, DIM), label0=1)
el, es, rc = one.topk_batch(qs, K)
assert rc == 0 and (labels == el).all() and scores.astype(np.float32).tobytes() == es.astype(np.float32).tobytes(), rank
L.VecSimB200_ShardGroup_Free(g)
dist.barrier()
if rank == 0: print("SHARDGROUP-WIDE-OK")
"""


@pytest.mark.gpu
def test_shard_group_of_two_ranks_at_k_1000(tmp_path):
    """Two processes, two GPUs (NCCL puts one rank on each device): the merged k = 1000 answer equals the single index over the
    whole corpus.  Skipped on a single-GPU box, where test_shard_groups_equal_the_single_index merges two shards' exchange
    blocks with the same merge kernel."""
    import subprocess
    import sys

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "sg_wide.py"
    script.write_text(f"ROOT = {root!r}\n" + _NCCL_WIDE)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29543", str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SHARDGROUP-WIDE-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
