"""KNN batches on multi-value indexes (a label owns several rows; its score is the minimum over them).  VecSimB200_TopKQueryBatch
and ..Device answer them on the device: a tensor-core route selects each query's K = min(128, k*m, n) best rows and the label
stage takes their first k distinct labels, proven when the K rows hold k of them; other queries, and batches no tensor-core route
serves, run the label-aware exact scan (DESIGN.md §4.4).  Every answer must equal the per-query VecSimIndex_TopKQuery on the same
index and the reference (the C restatement at the AVX-512 tier) with multi=True: ids and score bits for fp32 and the 8-bit
types, the 1e-2 bar for fp16 / bf16.
"""
import ctypes as C
import math

import numpy as np
import pytest

import oracle_lib as ol
from test_vecsim_parity import assert_same

SIZE_MAX = np.uint64(0xFFFFFFFFFFFFFFFF)
_KEEPALIVE = []  # ctypes trampolines must outlive their registration


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


# ------------------------------------------------------------------------------------------------------------------
# label layouts
# ------------------------------------------------------------------------------------------------------------------
def rows_per_label(shape, n, rng):
    """Row counts per label summing to n: "1", "3", "rand" (1..8), "skew" (one label of 300, the rest 2), or an int."""
    if shape == "rand":
        c = rng.integers(1, 9, n)
    elif shape == "skew":
        c = np.full(n, 2)
        c[0] = 300
    else:
        c = np.full(n, int(shape))
    cs = np.cumsum(c)
    nl = int(np.searchsorted(cs, n)) + 1
    c = c[:nl].copy()
    c[-1] -= int(cs[nl - 1]) - n
    assert c.sum() == n and (c > 0).all()
    return c


def make_labels(shape, n, rng, place):
    """Per-row labels (1-based, spaced by 3 so that label and row order differ); "contig" keeps a label's rows together,
    "scatter" spreads them over the index."""
    c = rows_per_label(shape, n, rng)
    lab = np.repeat(1 + 3 * np.arange(len(c), dtype=np.uint64), c)
    if place == "scatter":
        lab = lab[rng.permutation(n)]
    return lab


def chunk_rows(rng, n_labels, per, dim, spread=0.05):
    """"Chunks": per rows of each label near a per-label centre, contiguous.  fp32 rows, per-row labels."""
    centres = rng.standard_normal((n_labels, dim)).astype(np.float32)
    rows = np.repeat(centres, per, axis=0) + spread * rng.standard_normal((n_labels * per, dim)).astype(np.float32)
    labels = np.repeat(1 + np.arange(n_labels, dtype=np.uint64), per)
    return rows.astype(np.float32), labels, centres


# ------------------------------------------------------------------------------------------------------------------
# CPU: a numpy model of the selection proof and the per-list dedup
# ------------------------------------------------------------------------------------------------------------------
def _first_distinct(order, labels, k):
    out, seen = [], set()
    for r in order:
        lab = int(labels[r])
        if lab not in seen:
            seen.add(lab)
            out.append(int(r))
            if len(out) == k:
                break
    return out, len(seen)


def _list_model(rows_seen, comp, labels, k):
    """A label-aware list fed row by row: a listed label is replaced only by a smaller composite, a new one evicts the worst."""
    lst = {}  # label -> row
    for r in rows_seen:
        lab = int(labels[r])
        if lab in lst:
            if comp[r] < comp[lst[lab]]:
                lst[lab] = r
        elif len(lst) < k:
            lst[lab] = r
        else:
            worst = max(lst, key=lambda l: comp[lst[l]])
            if comp[r] < comp[lst[worst]]:
                del lst[worst]
                lst[lab] = r
    return list(lst.values())


def test_selection_proof_and_per_list_dedup_model():
    rng = np.random.default_rng(5)
    for trial in range(40):
        n = int(rng.integers(50, 400))
        labels = make_labels(["1", "3", "rand", "skew" if n > 320 else "rand"][trial % 4], n, rng, ["contig", "scatter"][trial % 2])
        scores = rng.integers(0, 30, n).astype(np.float64)  # planted ties: few distinct scores
        comp = scores * 1e6 + np.arange(n)                # the (score, row id) composite
        order = np.argsort(comp)
        n_labels = len(set(labels.tolist()))
        m = max(np.unique(labels, return_counts=True)[1])
        for k in (1, 3, 10, 40):
            kk = min(k, n_labels)
            truth, _ = _first_distinct(order, labels, kk)  # best row per label, labels by that row's composite
            best = {}
            for r in range(n):
                lab = int(labels[r])
                if lab not in best or comp[r] < comp[best[lab]]:
                    best[lab] = r
            brute = sorted(best.values(), key=lambda r: comp[r])[:kk]
            assert truth == brute
            for K in sorted({kk, min(n, 2 * kk), min(n, kk * m), min(n, 128), n}):
                sel, distinct = _first_distinct(order[:K], labels, kk)
                if distinct >= kk:  # the check
                    assert sel == brute, (trial, k, K)
                if K >= min(n, k * m):  # the guarantee
                    assert distinct >= kk
            # per-list dedup: rows dealt to lists in random order, each list label-aware, then the same rule on the union
            n_lists = int(rng.integers(1, 9))
            owner = rng.integers(0, n_lists, n)
            union = []
            for li in range(n_lists):
                mine = rng.permutation(np.flatnonzero(owner == li))
                union += _list_model(mine, comp, labels, kk)
            merged, _ = _first_distinct(sorted(union, key=lambda r: comp[r]), labels, kk)
            assert merged == brute, (trial, k, n_lists)


def test_chunk_builder_has_power():
    """On exact distances most "chunk" queries see fewer than k labels among their 128 best rows, so the label check fails and
    the label-aware exact scan has to answer them: the fallback test below exercises that path."""
    rng = np.random.default_rng(11)
    k = 10
    rows, labels, centres = chunk_rows(rng, 400, 50, 64)
    qs = centres[rng.integers(0, 400, 32)] + 0.05 * rng.standard_normal((32, 64)).astype(np.float32)
    r = rows / np.linalg.norm(rows, axis=1, keepdims=True)
    q = qs / np.linalg.norm(qs, axis=1, keepdims=True)
    d = 1.0 - q.astype(np.float64) @ r.T.astype(np.float64)
    few = 0
    for i in range(len(qs)):
        top = np.argsort(d[i], kind="stable")[:128]
        few += len(set(labels[top].tolist())) < k
    assert few >= 0.9 * len(qs), few


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
_VT = {ol.F32: 0, ol.BF16: 2, ol.F16: 3, ol.I8: 4, ol.U8: 5}
_MT = {ol.L2: 0, ol.IP: 1, ol.COS: 2}


def _pair(vtype, metric, dim, rows, labels):
    vs = _vs()
    g = vs.VecSimIndex(_VT[vtype], dim, _MT[metric], multi=True)
    p = ol.PortIndex(vtype, dim, metric, multi=True, tier=ol.TIER_AVX512)
    assert g.add_many(rows, labels=labels) == len(rows)
    for r, lab in zip(rows, labels.tolist()):
        p.add(r, lab)
    return g, p


def _rows(vtype, metric, seed, n, dim):
    rows = ol.synth_rows(vtype, seed, 0, n, dim)
    if vtype == ol.F32 and metric == ol.IP:  # raw inner product: keep 1 - dot away from the fp16 limits
        rows = (rows.astype(np.float64) / math.sqrt(dim)).astype(np.float32)
    return rows


def _check_host(g, p, qs, k, labels, scores, exact, metric):
    """Host API rows against the per-query call on the same index (identical) and the reference (ids and score bits for the
    exact types; in a run of exactly tied scores at the k-th label the reference keeps the smaller labels, this library the
    smaller row ids, DESIGN.md §3.2)."""
    for i in range(qs.shape[0]):
        gi, gs, code = g.topk(qs[i], k)
        assert code == 0
        h = int((labels[i] != SIZE_MAX).sum())
        assert (labels[i, h:] == SIZE_MAX).all() and np.isnan(scores[i, h:]).all()
        bi, bs = labels[i, :h].astype(np.int64), scores[i, :h]
        assert len(set(bi.tolist())) == h
        if exact:
            assert bi.tolist() == gi.tolist(), (i, bi[:12].tolist(), gi[:12].tolist())
            assert bs.astype(np.float32).tobytes() == gs.astype(np.float32).tobytes(), i
        else:
            assert_same(bi, bs, gi, gs, False, metric)
        pi, ps = p.topk(qs[i], k)
        if exact:
            assert bs.astype(np.float32).tobytes() == ps.astype(np.float32).tobytes(), i
            if h:
                below = bs.astype(np.float32) < np.float32(bs[-1])
                assert bi[below].tolist() == pi[below].tolist(), i
        else:
            assert_same(bi, bs, pi, ps, False, metric)


def _device_batch(g, qs, k):
    """The device API takes queries in stored form: cosine queries are normalised first (the library's own normalisation)."""
    import torch

    vs = _vs()
    nq = qs.shape[0]
    blob = g.dim * vs.ELEM_SIZE[g.vtype]
    stored = blob + (4 if g.metric == vs.VecSimMetric_Cosine and g.vtype in (vs.VecSimType_INT8, vs.VecSimType_UINT8) else 0)
    pitch = (stored + 15) // 16 * 16  # the device API reads query i at i * round16(stored bytes)
    buf = np.zeros((nq, pitch), dtype=np.uint8)
    buf[:, :blob] = np.ascontiguousarray(qs).view(np.uint8).reshape(nq, blob)
    if g.metric == vs.VecSimMetric_Cosine:  # int8 / uint8: the norm is appended after the payload
        for q in buf:
            vs.normalize(q, g.dim, g.vtype)
    qd = torch.from_numpy(buf).cuda()
    out_l = torch.full((max(nq, 1), max(k, 1)), 7, dtype=torch.int64, device="cuda")
    out_s = torch.zeros((max(nq, 1), max(k, 1)), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp)
    torch.cuda.synchronize()
    return rc, out_l.cpu().numpy(), out_s.cpu().numpy()


def _flags(g, nq):
    f = np.zeros(nq, dtype=np.uint32)
    assert _vs().lib().VecSimB200_LastCoarseFlags(g.h, f.ctypes.data, nq) == 0
    return f


def _device_equals_host(g, qs, k, dl, ds):
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0
    h = hl != SIZE_MAX
    assert ((dl >= 0) == h).all()
    assert (dl[h].astype(np.uint64) == hl[h]).all()
    assert ds[h].tobytes() == hs[h].astype(np.float32).tobytes()
    return hl, hs


# ------------------------------------------------------------------------------------------------------------------
# GPU: parity matrix (host API)
# ------------------------------------------------------------------------------------------------------------------
# (vtype, metric, dim, n, nq, k, rows per label, placement): every dtype / metric of the issue, every shape and placement,
# k in {1, 10, 100}, nq in {1, 16, 256}, n = 20k (exact route) and 70k / 300k (tensor-core routes)
_MATRIX = [
    (ol.F32, ol.COS, 128, 70_000, 256, 10, "3", "contig"),
    (ol.F32, ol.COS, 128, 300_000, 16, 100, "rand", "scatter"),
    (ol.F32, ol.COS, 96, 20_000, 16, 10, "skew", "scatter"),
    (ol.F32, ol.COS, 128, 70_000, 1, 10, "rand", "contig"),
    (ol.F32, ol.L2, 128, 70_000, 256, 100, "skew", "contig"),
    (ol.F32, ol.L2, 64, 20_000, 256, 1, "3", "scatter"),
    (ol.F32, ol.IP, 128, 70_000, 16, 1, "1", "scatter"),
    (ol.F32, ol.IP, 256, 300_000, 256, 10, "3", "scatter"),
    (ol.F16, ol.IP, 128, 70_000, 256, 10, "rand", "scatter"),
    (ol.F16, ol.IP, 64, 20_000, 16, 100, "3", "contig"),
    (ol.BF16, ol.COS, 128, 70_000, 16, 100, "skew", "scatter"),
    (ol.BF16, ol.COS, 128, 20_000, 1, 1, "rand", "scatter"),
    (ol.I8, ol.COS, 128, 70_000, 256, 100, "rand", "scatter"),
    (ol.I8, ol.COS, 96, 20_000, 16, 10, "1", "contig"),
    (ol.U8, ol.IP, 128, 70_000, 16, 10, "skew", "contig"),
    (ol.U8, ol.IP, 128, 300_000, 256, 1, "3", "scatter"),
    (ol.U8, ol.IP, 128, 20_000, 16, 10, "rand", "scatter"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,dim,n,nq,k,shape,place", _MATRIX)
def test_batch_matches_per_query_and_reference(vtype, metric, dim, n, nq, k, shape, place):
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(-1)
    rng = np.random.default_rng(n + dim + k + nq)
    labels = make_labels(shape, n, rng, place)
    g, p = _pair(vtype, metric, dim, _rows(vtype, metric, 42, n, dim), labels)
    qs = _rows(vtype, metric, 43, nq, dim)
    bl, bs, rc = g.topk_batch(qs, k)
    assert rc == 0
    tensor = n >= 65536 and nq >= 16
    assert vs.lib().VecSimB200_LastBatchPath(g.h) == ((2 if vtype != ol.F32 else 1) if tensor else 0)
    _check_host(g, p, qs, k, bl, bs, vtype not in (ol.F16, ol.BF16), metric)


# ------------------------------------------------------------------------------------------------------------------
# GPU: routes and flags through the device API
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_three_rows_per_label_stay_on_the_tensor_core_route():
    """m = 3, k = 10: K = 30 rows always hold 10 labels, so every query is proven on the row route (flags 1 or 2)."""
    vs = _vs()
    n, dim, nq, k = 70_000, 128, 256, 10
    labels = make_labels("3", n, np.random.default_rng(1), "scatter")
    g, p = _pair(ol.F32, ol.COS, dim, _rows(ol.F32, ol.COS, 42, n, dim), labels)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
    rc, dl, ds = _device_batch(g, qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    f = _flags(g, nq)
    assert np.isin(f, (1, 2)).all(), np.bincount(f, minlength=4).tolist()
    hl, hs = _device_equals_host(g, qs, k, dl, ds)
    _check_host(g, p, qs[::8], k, hl[::8], hs[::8], True, ol.COS)


@pytest.mark.gpu
def test_chunks_fall_back_to_the_label_aware_exact_scan():
    """50 rows per label near a centre: the 128 best rows of most queries hold fewer than 10 labels (flag 3); the label-aware
    exact scan answers those, still exactly."""
    vs = _vs()
    rng = np.random.default_rng(2)
    dim, nq, k = 64, 32, 10
    rows, labels, centres = chunk_rows(rng, 1600, 50, dim)
    g, p = _pair(ol.F32, ol.COS, dim, rows, labels)
    qs = (centres[rng.integers(0, 1600, nq)] + 0.05 * rng.standard_normal((nq, dim))).astype(np.float32)
    rc, dl, ds = _device_batch(g, qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    f = _flags(g, nq)
    assert (f == 3).sum() >= nq // 2, np.bincount(f, minlength=4).tolist()
    hl, hs = _device_equals_host(g, qs, k, dl, ds)
    _check_host(g, p, qs, k, hl, hs, True, ol.COS)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(ol.I8, ol.COS), (ol.F16, ol.IP)])
def test_chunks_after_the_direct_routes_fall_back_too(vtype, metric):
    """The same chunk shape on int8 and fp16 corpora: after the 8-bit / 16-bit direct routes most queries fail the label check
    (flag 3) and the label-aware exact scan answers them on the device: int8 exactly, fp16 within the 1e-2 bar."""
    vs = _vs()
    rng = np.random.default_rng(12)
    dim, nq, k, n_labels = 64, 32, 10, 1600
    centres = rng.uniform(-0.7, 0.7, (n_labels, dim)).astype(np.float32)
    x = np.repeat(centres, 50, axis=0) + 0.02 * rng.standard_normal((n_labels * 50, dim)).astype(np.float32)
    q = centres[rng.integers(0, n_labels, nq)] + 0.02 * rng.standard_normal((nq, dim)).astype(np.float32)
    if vtype == ol.I8:
        rows, qs = np.rint(127.0 * np.clip(x, -1, 1)).astype(np.int8), np.rint(127.0 * np.clip(q, -1, 1)).astype(np.int8)
    else:
        rows, qs = x.astype(np.float16).view(np.uint16), q.astype(np.float16).view(np.uint16)
    labels = np.repeat(1 + np.arange(n_labels, dtype=np.uint64), 50)
    g, p = _pair(vtype, metric, dim, rows, labels)
    rc, dl, ds = _device_batch(g, qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 2
    f = _flags(g, nq)
    assert (f == 3).sum() >= nq // 2, np.bincount(f, minlength=4).tolist()
    exact = vtype == ol.I8
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0
    for i in range(nq):
        gi, gs, _ = g.topk(qs[i], k)
        if exact:  # device API (label-aware exact scan) == host API == per-query call
            assert dl[i].tolist() == gi.tolist() and ds[i].tobytes() == gs.astype(np.float32).tobytes(), i
        else:
            assert_same(dl[i].astype(np.int64), ds[i].astype(np.float64), gi, gs, False, metric)
    _check_host(g, p, qs, k, hl, hs, exact, metric)


@pytest.mark.gpu
def test_wide_labels_cap_K_at_128_and_still_prove():
    """m = 20 scattered rows per label, k = 10: k * m = 200 > 128, so K = 128; random scattered rows put far more than 10 labels
    among any 128 rows, so the check passes."""
    vs = _vs()
    n, dim, nq, k = 70_000, 128, 64, 10
    labels = make_labels("20", n, np.random.default_rng(3), "scatter")
    g, p = _pair(ol.F32, ol.COS, dim, _rows(ol.F32, ol.COS, 42, n, dim), labels)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
    rc, dl, ds = _device_batch(g, qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    f = _flags(g, nq)
    assert np.isin(f, (1, 2)).all(), np.bincount(f, minlength=4).tolist()
    hl, hs = _device_equals_host(g, qs, k, dl, ds)
    _check_host(g, p, qs, k, hl, hs, True, ol.COS)


@pytest.mark.gpu
def test_near_duplicate_siblings_need_K_of_k_times_m():
    """Each label's 3 rows are near-duplicates, so a query's best rows come in sibling triples: 10 rows hold only 4 labels,
    30 rows hold 10.  With K = k * m every query is proven on the first tier (flag 1)."""
    vs = _vs()
    rng = np.random.default_rng(4)
    n_labels, dim, nq, k = 24_000, 128, 64, 10
    base = _rows(ol.F32, ol.COS, 42, n_labels, dim)
    rows = (np.repeat(base, 3, axis=0) + 1e-4 * rng.standard_normal((3 * n_labels, dim))).astype(np.float32)
    labels = np.repeat(1 + np.arange(n_labels, dtype=np.uint64), 3)
    g, p = _pair(ol.F32, ol.COS, dim, rows, labels)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
    rc, dl, ds = _device_batch(g, qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    f = _flags(g, nq)
    assert (f == 1).all(), np.bincount(f, minlength=4).tolist()
    hl, hs = _device_equals_host(g, qs, k, dl, ds)
    _check_host(g, p, qs, k, hl, hs, True, ol.COS)


# ------------------------------------------------------------------------------------------------------------------
# GPU: edge cases, updates, shards, timeouts
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [20_000, 70_000])
def test_k_beyond_the_label_count(n):
    """k > label_count: every label once, then empty slots (SIZE_MAX / NaN on the host API, -1 on the device API)."""
    dim, nq = 64, 16
    rng = np.random.default_rng(6)
    labels = (1 + rng.integers(0, 40, n)).astype(np.uint64)  # 40 labels of ~n/40 rows
    g, p = _pair(ol.F32, ol.COS, dim, _rows(ol.F32, ol.COS, 42, n, dim), labels)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
    bl, bs, rc = g.topk_batch(qs, 100)
    assert rc == 0 and ((bl != SIZE_MAX).sum(1) == 40).all()
    _check_host(g, p, qs, 100, bl, bs, True, ol.COS)
    rc, dl, ds = _device_batch(g, qs, 100)
    assert rc == 0 and (dl[:, 40:] == -1).all() and np.isnan(ds[:, 40:]).all()
    _device_equals_host(g, qs, 100, dl, ds)


@pytest.mark.gpu
def test_empty_index_and_empty_batches():
    vs = _vs()
    dim = 32
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
    qs = _rows(ol.F32, ol.COS, 43, 4, dim)
    bl, bs, rc = g.topk_batch(qs, 5)
    assert rc == 0 and (bl == SIZE_MAX).all() and np.isnan(bs).all()
    rc, dl, _ = _device_batch(g, qs, 5)
    assert rc == 0 and (dl == -1).all()
    g.add_many(_rows(ol.F32, ol.COS, 42, 100, dim), labels=np.repeat(np.arange(1, 51, dtype=np.uint64), 2))
    bl, bs, rc = g.topk_batch(qs[:0], 5)
    assert rc == 0 and bl.shape == (0, 5)
    bl, bs, rc = g.topk_batch(qs, 0)
    assert rc == 0 and bl.shape == (4, 0)
    assert _device_batch(g, qs[:0], 5)[0] == 0
    rc, dl, _ = _device_batch(g, qs, 0)
    assert rc == 0 and (dl == 7).all()  # nothing written


@pytest.mark.gpu
@pytest.mark.parametrize("n", [20_000, 70_000])
def test_updates_between_batches(n):
    """Rows appended to existing labels (m grows from 2 to 6), labels deleted (the swap-delete moves rows of other labels to new
    ids), then re-added: each batch equals the per-query call and the reference."""
    dim, nq, k = 64, 32, 10
    rng = np.random.default_rng(7)
    labels = make_labels("2", n, rng, "scatter")
    g, p = _pair(ol.F32, ol.L2, dim, _rows(ol.F32, ol.L2, 42, n, dim), labels)
    qs = _rows(ol.F32, ol.L2, 43, nq, dim)

    def check():
        bl, bs, rc = g.topk_batch(qs, k)
        assert rc == 0
        _check_host(g, p, qs, k, bl, bs, True, ol.L2)
        return bl

    first = check()
    grow = list(dict.fromkeys(int(x) for x in first[:, :3].ravel()))[:50]
    extra = _rows(ol.F32, ol.L2, 44, 4 * len(grow), dim)
    for i, lab in enumerate(np.repeat(grow, 4).tolist()):  # some of the best labels grow to 6 rows each
        assert g.add(extra[i], int(lab)) == 1 and p.add(extra[i], int(lab)) == 1
    check()
    gone = [int(x) for x in first[:8, :3].ravel()]
    for lab in set(gone):
        assert g.delete(lab) > 0 and p.delete(lab) > 0
    second = check()
    assert not set(gone) & set(second.ravel().tolist())
    for j, lab in enumerate(sorted(set(gone))):
        assert g.add(extra[j], lab) == 1 and p.add(extra[j], lab) == 1
    check()


@pytest.mark.gpu
def test_shard_group_of_one_and_two_label_disjoint_shards():
    """World 1: the collective entry point answers like the index.  Two shards that split the labels (a label's rows live on one
    shard, as RediSearch shards by document) merged with VecSimB200_MergeShardTopK equal one index."""
    import torch

    from redisearch_b200 import sharding

    vs = _vs()
    L = vs.lib()
    n, dim, nq, k = 70_000, 64, 32, 10
    rng = np.random.default_rng(8)
    labels = make_labels("rand", n, rng, "scatter")
    rows = _rows(ol.F32, ol.COS, 42, n, dim)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
    one, p = _pair(ol.F32, ol.COS, dim, rows, labels)
    el, es, rc = one.topk_batch(qs, k)
    assert rc == 0
    grp = L.VecSimB200_ShardGroup_New(None, 0, 1)
    assert grp
    gl = np.zeros((nq, k), dtype=np.uint64)
    gs = np.zeros((nq, k), dtype=np.float64)
    assert L.VecSimB200_ShardGroup_TopKBatch(grp, one.h, qs.ctypes.data, qs.strides[0], nq, k, gl.ctypes.data, gs.ctypes.data) == 0
    assert (gl == el).all() and gs.astype(np.float32).tobytes() == es.astype(np.float32).tobytes()
    L.VecSimB200_ShardGroup_Free(grp)
    side = (labels % np.uint64(2)).astype(bool)
    ss = np.zeros((2, nq, k), dtype=np.float32)
    sl = np.zeros((2, nq, k), dtype=np.int64)
    for s in range(2):
        sel = side == bool(s)
        ix = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
        assert ix.add_many(rows[sel], labels=labels[sel]) == int(sel.sum())
        rc, dl, ds = _device_batch(ix, qs, k)
        assert rc == 0
        sl[s], ss[s] = dl, ds
    ms, ml = sharding.merge_topk_device(torch.from_numpy(ss).cuda(), torch.from_numpy(sl).cuda())
    torch.cuda.synchronize()
    assert (ml.cpu().numpy() == el.astype(np.int64)).all()
    assert ms.cpu().numpy().tobytes() == es.astype(np.float32).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [20_000, 70_000])
def test_timeout_fires_at_once(n):
    vs = _vs()
    L = vs.lib()
    dim = 64
    labels = make_labels("3", n, np.random.default_rng(9), "contig")
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine, multi=True)
    g.add_many(_rows(ol.F32, ol.COS, 42, n, dim), labels=labels)
    qs = _rows(ol.F32, ol.COS, 43, 32, dim)
    cb, cb_off = vs.TIMEOUT_CB(lambda ctx: 1), vs.TIMEOUT_CB(lambda ctx: 0)
    _KEEPALIVE.extend([cb, cb_off])
    L.VecSim_SetTimeoutCallbackFunction(cb)
    try:
        qp = vs.VecSimQueryParams()
        _, _, rc = g.topk_batch(qs, 10, C.byref(qp))
        assert rc == vs.VecSim_QueryReply_TimedOut
    finally:
        L.VecSim_SetTimeoutCallbackFunction(cb_off)
    bl, bs, rc = g.topk_batch(qs, 10)
    assert rc == 0 and (bl != SIZE_MAX).all()


@pytest.mark.gpu
def test_timeout_while_the_label_aware_scan_runs():
    """A deadline that passes while the label-aware exact scan runs (a corpus below the tensor-core routes' 65,536 rows, so the
    host API scans every query): TimedOut at once, the scan's context is abandoned and drained, and the next batch is exact."""
    vs = _vs()
    L = vs.lib()
    n, dim, nq, k = 60_000, 256, 256, 100
    labels = make_labels("3", n, np.random.default_rng(13), "scatter")
    g, p = _pair(ol.F32, ol.COS, dim, _rows(ol.F32, ol.COS, 42, n, dim), labels)
    qs = _rows(ol.F32, ol.COS, 43, nq, dim)
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
    bl, bs, rc = g.topk_batch(qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 0
    _check_host(g, p, qs[::16], k, bl[::16], bs[::16], True, ol.COS)
