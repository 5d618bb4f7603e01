"""Sharded filtered KNN, range and filtered range batches: the counted exchange block, its device merge
(VecSimB200_MergeShardListBlocks) against a numpy model, shards merged against one index holding every row, and the
ShardGroup collectives (world = 1 on one GPU, two ranks over NCCL where two GPUs exist)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_SCORE, BY_ID = 0, 1
EMPTY_MODE, HYBRID_ADHOC_BF, HYBRID_BATCHES = 0, 2, 3
_VT = {ol.F32: 0, ol.F16: 3, ol.BF16: 2, ol.I8: 4, ol.U8: 5}
_MT = {ol.L2: 0, ol.IP: 1, ol.COS: 2}
FAILED = 0xFFFFFFFF
NAN_TOPW, NAN_RANGE = 0x7FC00000, 0x7FFFFFFF  # the pads of the KNN and range calls


def _lib():
    from redisearch_b200 import vecsim as vs

    return vs.lib()


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq,w", [(1, 1), (1, 10), (3, 7), (33, 1000), (256, 4096), (5, 3)])
def test_block_bytes_are_the_layout_padded_to_16(nq, w):
    b = int(_lib().VecSimB200_ShardListBlockBytes(nq, w))
    assert b % 16 == 0 and nq * w * 12 + nq * 4 <= b < nq * w * 12 + nq * 4 + 16


@pytest.mark.parametrize("G,nq,w,rng_kind,order", [
    (0, 4, 10, 0, BY_SCORE),            # no rank
    (2, 4, 0, 0, BY_SCORE),             # w == 0
    (2, 4, 4097, 1, BY_SCORE),          # w > 4096
    (2, (1 << 31) + 1, 10, 0, BY_SCORE),  # nq > 2^31
    (2, 4, 10, 2, BY_SCORE),            # unknown kind
    (2, 4, 10, 1, 2),                   # BY_SCORE_THEN_ID
    (2, 4, 10, 1, 7),                   # unknown order
    (2, 4, 10, 0, BY_ID),               # BY_ID with top-w
])
def test_merge_refusals_need_no_device(G, nq, w, rng_kind, order):
    assert _lib().VecSimB200_MergeShardListBlocks(None, G, nq, w, rng_kind, order, None, None, None, None) == -1


# ------------------------------------------------------------------------------------------------------------------
# the merge against a numpy model
# ------------------------------------------------------------------------------------------------------------------
def _okey(scores):
    """orderable_key of topk_common.cuh: -0.0 ties +0.0, NaN after +inf"""
    u = (scores.astype(np.float32) + np.float32(0)).view(np.uint32).astype(np.uint64)
    k = np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)
    return np.where(np.isnan(scores), 0xFFFFFFFE, k).astype(np.uint64)


SCORE_SET = np.array([-1.5, -0.0, 0.0, 0.25, 0.5, 1.0, 3.0], dtype=np.float32)


def _synth_blocks(G, nq, w, range_query, order, seed):
    """Per rank [nq, w] sorted runs in the local calls' order, their counts, each query one scenario: short runs, full runs,
    totals at w and w + 1, a rank over its cap, saturating counts, a failed rank, nothing at all"""
    rng = np.random.default_rng(seed)
    counts = np.zeros((G, nq), dtype=np.uint64)
    n_sc = 7 if range_query else 4
    for q in range(nq):
        sc = (q + seed) % n_sc
        if sc == 0:  # short runs
            counts[:, q] = rng.integers(0, w // max(G, 1) + 2, G) if range_query else rng.integers(0, w + 1, G)
        elif sc == 1:  # range: total exactly w; top-w: full runs
            counts[:, q] = rng.multinomial(w, np.ones(G) / G) if range_query else w
        elif sc == 2:  # range: total w + 1; top-w: a failed rank
            if range_query:
                counts[:, q] = rng.multinomial(w + 1, np.ones(G) / G)
            else:
                counts[:, q] = rng.integers(0, w + 1, G)
                counts[rng.integers(G), q] = FAILED
        elif sc == 3:  # nothing
            pass
        elif sc == 4:  # a rank over its cap
            counts[:, q] = rng.integers(0, 2, G)
            counts[rng.integers(G), q] = w + 1 + rng.integers(0, 5)
        elif sc == 5:  # counts whose sum saturates (G == 1: the largest real count)
            counts[:, q] = 0x80000000 if G > 1 else 0xFFFFFFFE
        else:  # a failed rank among answered ones
            counts[:, q] = rng.integers(0, 3, G)
            counts[rng.integers(G), q] = FAILED
    m = np.minimum(counts, w).astype(np.int64)
    m[counts == FAILED] = 0
    if range_query:
        m[counts > w] = 0  # a row over its cap is all -1
    scores = np.where(rng.random((G, nq, w)) < 0.6, SCORE_SET[rng.integers(0, len(SCORE_SET), (G, nq, w))],
                      rng.standard_normal((G, nq, w)).astype(np.float32)).astype(np.float32)
    labels = rng.integers(0, max(8, 2 * G * w), (G, nq, w)).astype(np.int64)  # duplicates across ranks: ties by rank
    key = _okey(scores)
    pri, sec = (labels.astype(np.uint64), key) if order == BY_ID else (key, labels.astype(np.uint64))
    grp = np.broadcast_to(np.arange(G * nq).reshape(G, nq, 1), (G, nq, w)).reshape(-1)
    idx = np.lexsort((sec.reshape(-1), pri.reshape(-1), grp))
    labels, scores = labels.reshape(-1)[idx].reshape(G, nq, w), scores.reshape(-1)[idx].reshape(G, nq, w)
    live = np.arange(w)[None, None, :] < m[:, :, None]
    labels = np.where(live, labels, -1)
    scores = np.where(live, scores, np.float32(np.nan)).astype(np.float32)
    return labels, scores, counts.astype(np.uint32)


def _model(labels, scores, counts, w, range_query, order):
    G, nq, _ = labels.shape
    c = counts.astype(np.uint64)
    failed = (c == FAILED).any(axis=0)
    total = c.sum(axis=0)
    m = np.minimum(c, w)
    merged = m.sum(axis=0)
    pad = NAN_RANGE if range_query else NAN_TOPW
    out_l = np.full((nq, w), -1, dtype=np.int64)
    out_s = np.full((nq, w), pad, dtype=np.uint32)
    out_c = np.where(failed, FAILED, np.minimum(total, FAILED) if range_query else np.minimum(total, w)).astype(np.uint32)
    blank = failed | ((total > w) if range_query else False)
    gg, qq, pp = np.nonzero(np.arange(w)[None, None, :] < m[:, :, None].astype(np.int64))
    keep = ~blank[qq]
    gg, qq, pp = gg[keep], qq[keep], pp[keep]
    lab = labels[gg, qq, pp]
    key = _okey(scores[gg, qq, pp])
    pri, sec = (lab.astype(np.uint64), key) if order == BY_ID else (key, lab.astype(np.uint64))
    idx = np.lexsort((pp, gg, sec, pri, qq))
    qs = qq[idx]
    start = np.searchsorted(qs, np.arange(nq))
    pos = np.arange(len(qs)) - start[qs]
    sel = pos < w
    out_l[qs[sel], pos[sel]] = lab[idx][sel]
    out_s[qs[sel], pos[sel]] = scores[gg, qq, pp][idx][sel].view(np.uint32)
    return out_l, out_s, out_c


def _merge(labels, scores, counts, range_query, order):
    import torch

    from redisearch_b200 import sharding

    parts = [(torch.from_numpy(labels[g]).cuda(), torch.from_numpy(scores[g]).cuda(), torch.from_numpy(counts[g].view(np.int32)).cuda())
             for g in range(labels.shape[0])]
    ol_, os_, oc = sharding.merge_shard_lists(parts, range_query=range_query, order=order)
    torch.cuda.synchronize()
    return ol_.cpu().numpy(), os_.cpu().numpy().view(np.uint32), oc.cpu().numpy().view(np.uint32)


KINDS = [(False, BY_SCORE), (True, BY_SCORE), (True, BY_ID)]
MERGE_SHAPES = [(G, nq, w) for G in (1, 2, 3, 8, 64) for w in (1, 10, 1000, 4096) for nq in (1, 33, 256) if G * nq * w <= 1 << 22]


@pytest.mark.gpu
@pytest.mark.parametrize("range_query,order", KINDS)
@pytest.mark.parametrize("G,nq,w", MERGE_SHAPES)
def test_merge_matches_the_model(G, nq, w, range_query, order):
    labels, scores, counts = _synth_blocks(G, nq, w, range_query, order, seed=G * 131 + nq * 7 + w)
    got = _merge(labels, scores, counts, range_query, order)
    exp = _model(labels, scores, counts, w, range_query, order)
    assert (got[2] == exp[2]).all(), np.nonzero(got[2] != exp[2])
    assert (got[0] == exp[0]).all(), np.nonzero((got[0] != exp[0]).any(axis=1))
    assert (got[1] == exp[1]).all(), np.nonzero((got[1] != exp[1]).any(axis=1))


@pytest.mark.gpu
def test_signed_zeros_tie_and_break_by_label_then_rank():
    """-0.0 and +0.0 are one key, as orderable_key makes them for the local calls; ties break by label, then by rank; score bits
    travel unchanged"""
    w = 6
    labels = np.array([[[3, 5, 9, -1, -1, -1]], [[4, 5, 8, -1, -1, -1]]], dtype=np.int64)
    scores = np.array([[[-0.0, 0.0, 0.0, np.nan, np.nan, np.nan]], [[0.0, -0.0, -0.0, np.nan, np.nan, np.nan]]], dtype=np.float32)
    counts = np.array([[3], [3]], dtype=np.uint32)
    gl, gs, gc = _merge(labels, scores, counts, False, BY_SCORE)
    assert gl[0].tolist() == [3, 4, 5, 5, 8, 9] and int(gc[0]) == 6
    assert gs[0].tolist() == np.array([-0.0, 0.0, 0.0, -0.0, -0.0, 0.0], dtype=np.float32).view(np.uint32).tolist()


# ------------------------------------------------------------------------------------------------------------------
# shards merged == one index
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mode1():
    L = _lib()
    L.VecSimB200_SetCoarseMode(1)
    yield L
    L.VecSimB200_SetCoarseMode(-1)


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cur():
    """torch's current stream: every library call of these tests is enqueued on it, so the copies and reads torch makes of the
    outputs are ordered after the calls whichever stream the process has made current"""
    import torch

    return torch.cuda.current_stream()


def _ok(r):
    """a device batch call's return tuple, its code checked"""
    assert r[-1] == 0, r[-1]
    return r


def _stage(ix, qs):
    from redisearch_b200 import vecsim as vs

    pitch = ix.query_pitch()
    buf = np.zeros((len(qs), pitch), dtype=np.uint8)
    for i in range(len(qs)):
        raw = np.ascontiguousarray(qs[i]).view(np.uint8)
        buf[i, :raw.size] = raw
        if ix.metric == vs.VecSimMetric_Cosine:
            vs.normalize(buf[i], ix.dim, ix.vtype)
    return _dev(buf)


def _params(policy):
    from redisearch_b200 import vecsim as vs

    if policy is None:
        return None
    p = vs.VecSimQueryParams()
    p.searchMode = policy
    return p


class Filters:
    """device buffers of ascending docId lists, with count pointers"""

    def __init__(self, filters):
        self.keep, self.ptrs, self.cptrs, self.caps = [], [], [], []
        for f in filters:
            buf, cnt = _dev(np.append(np.asarray(f, np.uint32), np.uint32(0)).view(np.int32)), _dev(np.array([len(f)], np.int32))
            self.keep += [buf, cnt]
            self.ptrs.append(buf.data_ptr() if len(f) else None)
            self.cptrs.append(cnt.data_ptr())
            self.caps.append(len(f))


class Corpus:
    """N docIds; single-value: row i is docId i + 1; multi-value: rows 2i, 2i + 1 are docId i + 1.  Shard g owns docIds
    sharding.doc_range(N, G, g) (lo, hi] with their rows; `empty_last`: the last shard holds nothing, the others split N."""

    def __init__(self, vtype, metric, n_docs, dim, multi=False, seed=42):
        self.vtype, self.metric, self.n, self.dim, self.multi = vtype, metric, n_docs, dim, multi
        self.rpd = 2 if multi else 1
        self.rows = ol.synth_rows(vtype, seed, 0, n_docs * self.rpd, dim)

    def index(self, lo, hi):
        from redisearch_b200 import vecsim as vs

        ix = vs.VecSimIndex(_VT[self.vtype], self.dim, _MT[self.metric], multi=self.multi)
        if hi > lo:
            labels = np.arange(lo * self.rpd, hi * self.rpd, dtype=np.uint64) // self.rpd + 1
            assert ix.add_many(self.rows[lo * self.rpd:hi * self.rpd], labels=labels) == (hi - lo) * self.rpd
        return ix

    def ranges(self, G, empty_last=False):
        from redisearch_b200 import sharding

        if empty_last:
            return [sharding.doc_range(self.n, G - 1, g) for g in range(G - 1)] + [(self.n, self.n)]
        return [sharding.doc_range(self.n, G, g) for g in range(G)]


def _slice(filters, lo, hi):
    from redisearch_b200 import sharding

    return [sharding.split_posting_list(np.asarray(f, np.uint32), None, lo, hi)[0] for f in filters]


def _host(t):
    lab, sc, cnt = t[:3]
    return lab.cpu().numpy(), sc.cpu().numpy().view(np.uint32), cnt.cpu().numpy().view(np.uint32)


def _assert_same(got, exp):
    gl, gs, gc = got
    el, es, ec = exp
    assert gc.tolist() == ec.tolist(), np.nonzero(gc != ec)
    bad = np.nonzero((gl != el).any(axis=1) | (gs != es).any(axis=1))[0]
    assert len(bad) == 0, (bad[:5].tolist(), gl[bad[0], :6].tolist(), el[bad[0], :6].tolist())


def _filters(rng, n, nq, fracs, ranges=None):
    """ascending docId lists over 1..n + 50 (the tail absent); fracs cycle per query: 0 = empty, 1 = every docId; a tuple gives
    the fraction per shard range (a batch whose shards see different filter widths)"""
    out = []
    for i in range(nq):
        fr = fracs[i % len(fracs)]
        if isinstance(fr, tuple):
            parts = [np.arange(lo + 1, hi + 1)[rng.random(hi - lo) < f] for f, (lo, hi) in zip(fr, ranges)]
            out.append(np.concatenate(parts).astype(np.uint32))
        elif fr >= 1:
            out.append(np.arange(1, n + 51, dtype=np.uint32))
        else:
            out.append(np.nonzero(rng.random(n + 50) < fr)[0].astype(np.uint32) + 1)
    return out


def _knn_radii(full, qs, rank):
    """per query the rank-th label distance over the whole corpus (rank <= 1000; multi-value: <= 128), a radius with about `rank`
    labels inside"""
    kk = min(rank, 128 if full.multi else 1000)
    _, scores, rc = full.topk_batch(qs, kk)
    assert rc == 0
    return _dev(scores[:, kk - 1].astype(np.float32))


def _sharded_hybrid_knn(corpus, G, qs, k, filters, policy=None, empty_last=False):
    from redisearch_b200 import sharding

    full = corpus.index(0, corpus.n)
    qd = _stage(full, qs)
    fl = Filters(filters)
    exp = _host(_ok(full.hybrid_topk_batch_device(qd, k, fl.ptrs, fl.caps, counts=fl.cptrs, params=_params(policy), stream=_cur())))
    parts, modes, keep = [], [], []
    for lo, hi in corpus.ranges(G, empty_last):
        ix = corpus.index(lo, hi)
        f = Filters(_slice(filters, lo, hi))
        lab, sc, cnt, md, rc = ix.hybrid_topk_batch_device(qd, k, f.ptrs, f.caps, counts=f.cptrs, params=_params(policy), stream=_cur())
        assert rc == 0, rc
        parts.append((lab, sc, cnt))
        modes.append(md)
        keep += [ix, f]
    got = _host(sharding.merge_shard_lists(parts))
    return got, exp, modes


def _sharded_range(corpus, G, qs, radii_rank, cap, order, filters=None, policy=None, empty_last=False):
    """label range (filters None) or hybrid range batches, sharded and merged, against the one index"""
    from redisearch_b200 import sharding

    full = corpus.index(0, corpus.n)
    qd = _stage(full, qs)
    rd = _knn_radii(full, qs, radii_rank)

    def call(ix, flt):
        if flt is None:
            r = ix.label_range_batch_device(qd, rd, cap, order, stream=_cur())
            assert r[3] == 0, r[3]
            return r[:3]
        f = Filters(flt)
        r = ix.hybrid_range_batch_device(qd, rd, cap, f.ptrs, f.caps, counts=f.cptrs, order=order, params=_params(policy), stream=_cur())
        assert r[4] == 0, r[4]
        return r[:3] + (f,)

    exp = _host(call(full, filters))
    parts, paths, keep = [], [], []
    for lo, hi in corpus.ranges(G, empty_last):
        ix = corpus.index(lo, hi)
        r = call(ix, None if filters is None else _slice(filters, lo, hi))
        parts.append(r[:3])
        paths.append(_lib().VecSimB200_LastBatchPath(ix.h))
        keep += [ix, r]
    got = _host(sharding.merge_shard_lists(parts, range_query=True, order=order))
    return got, exp, paths


FRACS = [0, 1e-4, 0.001, 0.01, 0.1, 0.5, 1.0]


@pytest.mark.gpu
@pytest.mark.parametrize("metric,G", [(ol.COS, 2), (ol.L2, 3)])
def test_hybrid_knn_fp32_dense_and_gather_shards_equal_one_index(mode1, metric, G):
    """>= 65,536 rows per shard: broad filters take the dense route on every shard, narrow ones the gather; k up to 1024"""
    rng = np.random.default_rng(G)
    corpus = Corpus(ol.F32, metric, 66_000 * G, 64)
    nq = 32
    qs = ol.synth_rows(ol.F32, 7, 0, nq, 64)
    filters = _filters(rng, corpus.n, nq, FRACS)
    for k, policy in ((10, None), (10, HYBRID_BATCHES), (100, None), (1024, HYBRID_ADHOC_BF), (1024, None)):
        got, exp, modes = _sharded_hybrid_knn(corpus, G, qs, k, filters, policy)
        _assert_same(got, exp)
        if policy == HYBRID_BATCHES:
            assert all((m == HYBRID_BATCHES).any() for m in modes), "a shard never took the dense route"


@pytest.mark.gpu
def test_hybrid_knn_one_shard_dense_the_other_gather(mode1):
    rng = np.random.default_rng(5)
    corpus = Corpus(ol.F32, ol.COS, 140_000, 64)
    nq = 24
    qs = ol.synth_rows(ol.F32, 8, 0, nq, 64)
    ranges = corpus.ranges(2)
    filters = _filters(rng, corpus.n, nq, [(0.6, 0.0005), (0.8, 0.001)], ranges)
    got, exp, modes = _sharded_hybrid_knn(corpus, 2, qs, 10, filters)
    _assert_same(got, exp)
    assert (modes[0] == HYBRID_BATCHES).any() and (modes[1] == HYBRID_ADHOC_BF).all(), modes


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,multi,G,empty_last", [
    (ol.I8, ol.L2, False, 2, False), (ol.U8, ol.L2, False, 3, False), (ol.F16, ol.IP, False, 3, False),
    (ol.BF16, ol.L2, False, 4, False), (ol.F32, ol.COS, True, 2, False), (ol.I8, ol.COS, True, 3, True),
    (ol.F32, ol.L2, False, 3, True)])
def test_hybrid_knn_other_types_shards_equal_one_index(mode1, vtype, metric, multi, G, empty_last):
    rng = np.random.default_rng(G + 10 * vtype)
    corpus = Corpus(vtype, metric, 20_000, 64, multi=multi)
    nq = 21
    qs = ol.synth_rows(vtype, 9, 0, nq, 64)
    filters = _filters(rng, corpus.n, nq, FRACS)
    for k in (1, 10, 128):
        got, exp, _ = _sharded_hybrid_knn(corpus, G, qs, k, filters, empty_last=empty_last)
        _assert_same(got, exp)


RANGE_VARIANTS = [  # vtype, metric, multi, docs, G: >= 65,536 rows per shard where the tensor-core routes should run
    (ol.F32, ol.COS, False, 132_000, 2), (ol.F32, ol.L2, False, 198_000, 3),
    (ol.I8, ol.L2, False, 132_000, 2), (ol.U8, ol.L2, False, 264_000, 4),
    (ol.F16, ol.IP, False, 30_000, 3), (ol.BF16, ol.L2, False, 30_000, 2),
    (ol.F32, ol.COS, True, 30_000, 3), (ol.U8, ol.COS, True, 30_000, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,multi,n,G", RANGE_VARIANTS)
def test_range_shards_equal_one_index(mode1, vtype, metric, multi, n, G):
    corpus = Corpus(vtype, metric, n, 64, multi=multi)
    nq = 32
    qs = ol.synth_rows(vtype, 11, 0, nq, 64)
    for rank, cap, order in ((50, 4096, BY_SCORE), (1000, 1000, BY_ID), (1000, 999, BY_SCORE), (1000, 256, BY_ID), (1, 1, BY_ID)):
        got, exp, paths = _sharded_range(corpus, G, qs, rank, cap, order)
        _assert_same(got, exp)
        if n // G >= 65_536 and not multi:  # every shard on its tensor-core route: fp32 (1) or 8-bit (2)
            assert paths == [1 if vtype == ol.F32 else 2] * G, paths


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,multi,n,G,empty_last", [
    (ol.F32, ol.COS, False, 132_000, 2, False), (ol.I8, ol.L2, False, 132_000, 2, False), (ol.F16, ol.L2, False, 20_000, 3, False),
    (ol.F32, ol.IP, True, 20_000, 3, False), (ol.U8, ol.L2, False, 40_000, 3, True)])
def test_hybrid_range_shards_equal_one_index(mode1, vtype, metric, multi, n, G, empty_last):
    rng = np.random.default_rng(n + G)
    corpus = Corpus(vtype, metric, n, 64, multi=multi)
    nq = 28
    qs = ol.synth_rows(vtype, 12, 0, nq, 64)
    filters = _filters(rng, corpus.n, nq, FRACS)
    for rank, cap, order, policy in ((1000, 4096, BY_SCORE, None), (1000, 64, BY_ID, None), (1000, 4096, BY_SCORE, HYBRID_BATCHES),
                                     (500, 300, BY_ID, HYBRID_ADHOC_BF)):
        got, exp, paths = _sharded_range(corpus, G, qs, rank, cap, order, filters=filters, policy=policy, empty_last=empty_last)
        _assert_same(got, exp)
        if policy == HYBRID_BATCHES and n // G >= 65_536 and not multi:
            assert paths == [1 if vtype == ol.F32 else 2] * G, paths


@pytest.mark.gpu
def test_pending_device_filters_feed_every_shard(mode1):
    """each shard's AND / OR of its posting-list slices, from II_IntersectBatchDevice / II_UnionBatchDevice, is fed while still
    pending; the merged rows equal the one index's over the whole lists"""
    from redisearch_b200 import postings as ps
    from redisearch_b200 import sharding

    rng = np.random.default_rng(31)
    G, n, nq, k = 2, 140_000, 16, 10
    corpus = Corpus(ol.F32, ol.COS, n, 64)
    pool = [np.sort(rng.choice(np.arange(1, n + 1), s, replace=False)).astype(np.uint64) for s in (90_000, 70_000, 3_000)]
    qs = ol.synth_rows(ol.F32, 13, 0, nq, 64)
    full = corpus.index(0, n)
    qd = _stage(full, qs)
    rd = _knn_radii(full, qs, 500)
    shards = [(lo, hi, corpus.index(lo, hi)) for lo, hi in corpus.ranges(G)]
    for kind in ("and", "or"):
        batch_fn = ps.intersect_batch_device if kind == "and" else ps.union_batch_device
        set_fn = np.intersect1d if kind == "and" else np.union1d
        filters = [set_fn(pool[i % 3], pool[(i + 1) % 3]).astype(np.uint32) for i in range(nq)]
        fl = Filters(filters)
        exp_knn = _host(_ok(full.hybrid_topk_batch_device(qd, k, fl.ptrs, fl.caps, counts=fl.cptrs, stream=_cur())))
        exp_rng = _host(_ok(full.hybrid_range_batch_device(qd, rd, 4096, fl.ptrs, fl.caps, counts=fl.cptrs, stream=_cur())))
        knn_parts, rng_parts, pending = [], [], []
        for lo, hi, ix in shards:
            pls = [ps.PostingList.from_arrays(sharding.split_posting_list(p, None, lo, hi)[0]) for p in pool]
            res = batch_fn([[pls[i % 3], pls[(i + 1) % 3]] for i in range(nq)], stream=_cur())
            ids, cnts, caps = [r[1] for r in res], [r[2] for r in res], [r[3] for r in res]
            lab, sc, cnt, _, rc = ix.hybrid_topk_batch_device(qd, k, ids, caps, counts=cnts, stream=_cur())
            assert rc == 0
            knn_parts.append((lab, sc, cnt))
            lab, sc, cnt, _, rc = ix.hybrid_range_batch_device(qd, rd, 4096, ids, caps, counts=cnts, stream=_cur())
            assert rc == 0
            rng_parts.append((lab, sc, cnt))
            pending.append((pls, res))
        _assert_same(_host(sharding.merge_shard_lists(knn_parts)), exp_knn)
        _assert_same(_host(sharding.merge_shard_lists(rng_parts, range_query=True)), exp_rng)
        for _, res in pending:
            for r in res:
                if r[0] is not None:
                    r[0].free_after(_cur())


# ------------------------------------------------------------------------------------------------------------------
# the collectives at world = 1
# ------------------------------------------------------------------------------------------------------------------
def _cp(ptrs):
    n = max(1, len(ptrs))
    return (C.c_void_p * n)(*[int(p) if p else None for p in ptrs])


def _collective(L, g, ix, kind, qd, nq, w, rd=None, order=BY_SCORE, fl=None, policy=None, stream=None, outs=None):
    """one ShardGroup list collective into torch outputs; returns (labels, scores, counts, modes, rc)"""
    import torch

    if outs is None:
        outs = (torch.empty((nq, w), dtype=torch.int64, device="cuda"), torch.empty((nq, w), dtype=torch.float32, device="cuda"),
                torch.empty(nq, dtype=torch.int32, device="cuda"))
    lab, sc, cnt = outs
    modes = np.zeros(max(1, nq), dtype=np.int32)
    sp = C.c_void_p((stream if stream is not None else _cur()).cuda_stream or None)
    p = _params(policy)
    pp = C.byref(p) if p is not None else None
    if kind == "knn":
        rc = L.VecSimB200_ShardGroup_HybridTopKBatchDevice(g, ix.h, qd.data_ptr(), nq, w, _cp(fl.ptrs), _cp(fl.cptrs),
                                                           (C.c_size_t * max(1, nq))(*fl.caps), pp, lab.data_ptr(), sc.data_ptr(),
                                                           cnt.data_ptr(), modes.ctypes.data, sp)
    elif kind == "range":
        rc = L.VecSimB200_ShardGroup_RangeQueryBatchDevice(g, ix.h, qd.data_ptr(), nq, rd.data_ptr(), w, order, lab.data_ptr(),
                                                           sc.data_ptr(), cnt.data_ptr(), sp)
    else:
        rc = L.VecSimB200_ShardGroup_HybridRangeQueryBatchDevice(g, ix.h, qd.data_ptr(), nq, rd.data_ptr(), w, order, _cp(fl.ptrs),
                                                                 _cp(fl.cptrs), (C.c_size_t * max(1, nq))(*fl.caps), pp, lab.data_ptr(),
                                                                 sc.data_ptr(), cnt.data_ptr(), modes.ctypes.data, sp)
    return lab, sc, cnt, modes[:nq], rc


@pytest.mark.gpu
def test_group_of_one_is_the_local_call(mode1):
    """world = 1: each collective equals its local call, launches exactly what the local call launches, and once the index is
    flushed returns while the caller's stream is still busy"""
    import torch

    L = mode1
    rng = np.random.default_rng(3)
    corpus = Corpus(ol.F32, ol.COS, 70_000, 64)
    ix = corpus.index(0, corpus.n)
    nq = 16
    qs = ol.synth_rows(ol.F32, 14, 0, nq, 64)
    qd = _stage(ix, qs)
    rd = _knn_radii(ix, qs, 300)
    fl = Filters(_filters(rng, corpus.n, nq, [0.001, 0.5]))
    g = L.VecSimB200_ShardGroup_New(None, 0, 1)
    assert g
    try:
        for kind, policy in (("knn", HYBRID_ADHOC_BF), ("knn", HYBRID_BATCHES), ("range", None), ("hybrid_range", HYBRID_ADHOC_BF),
                             ("hybrid_range", HYBRID_BATCHES)):
            w = 10 if kind == "knn" else 512

            def local():
                if kind == "knn":
                    return ix.hybrid_topk_batch_device(qd, w, fl.ptrs, fl.caps, counts=fl.cptrs, params=_params(policy), stream=_cur())
                if kind == "range":
                    return ix.label_range_batch_device(qd, rd, w, stream=_cur())
                return ix.hybrid_range_batch_device(qd, rd, w, fl.ptrs, fl.caps, counts=fl.cptrs, params=_params(policy), stream=_cur())

            exp = local()
            assert exp[-1] == 0
            exp = _host(exp)
            ix.stats(reset=True)
            local()
            want_launches = ix.stats(reset=True).kernel_launches
            got = _collective(L, g, ix, kind, qd, nq, w, rd=rd, fl=fl, policy=policy)
            launches = ix.stats(reset=True).kernel_launches
            assert got[4] == 0
            _assert_same(_host(got), exp)
            assert launches == want_launches, (kind, policy, launches, want_launches)
            # no host wait
            s = torch.cuda.Stream()
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(200_000_000)
            got2 = _collective(L, g, ix, kind, qd, nq, w, rd=rd, fl=fl, policy=policy, stream=s)
            busy = not s.query()
            s.synchronize()
            assert got2[4] == 0 and busy, "the call waited for the caller's stream"
            _assert_same(_host(got2), exp)
        # refusals of the shared arguments
        assert _collective(L, g, ix, "knn", qd, nq, 1025, fl=fl)[4] == -1
        assert _collective(L, g, ix, "range", qd, nq, 4097, rd=rd)[4] == -1
        assert _collective(L, g, ix, "hybrid_range", qd, nq, 64, rd=rd, order=2, fl=fl)[4] == -1
        assert _collective(L, g, ix, "knn", qd, nq, 10, fl=fl, policy=5)[4] == -1
    finally:
        L.VecSimB200_ShardGroup_Free(g)


# ------------------------------------------------------------------------------------------------------------------
# two ranks over NCCL
# ------------------------------------------------------------------------------------------------------------------
NCCL_SCRIPT = r'''
import os, sys, ctypes as C
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol
import test_vecsim_sharded_lists as T
from redisearch_b200 import vecsim as vs, sharding
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("gloo")          # control plane only: ships the 128-byte NCCL id
L = vs.lib()
L.VecSimB200_SetCoarseMode(1)
idbuf = np.zeros(128, dtype=np.uint8)
if rank == 0:
    assert L.VecSimB200_ShardGroup_UniqueId(idbuf.ctypes.data) == 0
t = torch.from_numpy(idbuf); dist.broadcast(t, 0)
g = L.VecSimB200_ShardGroup_New(idbuf.ctypes.data, rank, world)
assert g, "ncclCommInitRank failed"
corpus = T.Corpus(ol.F32, ol.COS, 140_000, 64)
lo, hi = sharding.doc_range(corpus.n, world, rank)
ix = corpus.index(lo, hi)
full = corpus.index(0, corpus.n)
nq = 24
qs = ol.synth_rows(ol.F32, 15, 0, nq, 64)
qd = T._stage(full, qs)
rd = T._knn_radii(full, qs, 400)
filters = T._filters(np.random.default_rng(1), corpus.n, nq, T.FRACS)
fl_all, fl_mine = T.Filters(filters), T.Filters(T._slice(filters, lo, hi))
for kind, w in (("knn", 10), ("knn", 1024), ("range", 4096), ("hybrid_range", 512)):
    for rep in range(2):
        got = T._collective(L, g, ix, kind, qd, nq, w, rd=rd, fl=fl_mine)
        assert got[4] == 0, (rank, kind, got[4])
    torch.cuda.synchronize()
    if kind == "knn":
        exp = full.hybrid_topk_batch_device(qd, w, fl_all.ptrs, fl_all.caps, counts=fl_all.cptrs, stream=T._cur())
    elif kind == "range":
        exp = full.label_range_batch_device(qd, rd, w, stream=T._cur())
    else:
        exp = full.hybrid_range_batch_device(qd, rd, w, fl_all.ptrs, fl_all.caps, counts=fl_all.cptrs, stream=T._cur())
    T._ok(exp)
    T._assert_same(T._host(got), T._host(exp))
# a rank whose local call refuses (-2: a filter cap beyond the 32-bit id range) still takes part; every row comes out failed
bad = T.Filters(T._slice(filters, lo, hi))
if rank == 1:
    bad.caps[0] = 0xFFFFFFF8
got = T._collective(L, g, ix, "knn", qd, nq, 10, fl=bad)
torch.cuda.synchronize()
assert got[4] == (-2 if rank == 1 else 0), (rank, got[4])
lab, sc, cnt = T._host(got)
assert (cnt == 0xFFFFFFFF).all() and (lab == -1).all(), rank
# and the group keeps working after it
got = T._collective(L, g, ix, "range", qd, nq, 4096, rd=rd)
torch.cuda.synchronize()
assert got[4] == 0
T._assert_same(T._host(got), T._host(T._ok(full.label_range_batch_device(qd, rd, 4096, stream=T._cur()))))
L.VecSimB200_ShardGroup_Free(g)
dist.barrier()
if rank == 0: print("SHARDLISTS-NCCL-OK")
'''


@pytest.mark.gpu
def test_list_collectives_over_nccl_two_ranks(tmp_path):
    """Two processes, two GPUs: the three collectives with ONE ncclAllGather inside the library each, every rank's merged rows
    equal to one index over the whole corpus; a rank refusing with -2 leaves no rank waiting.  Skipped on a single-GPU box."""
    import subprocess
    import sys

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "sl.py"
    script.write_text(f"ROOT = {ROOT!r}\n" + NCCL_SCRIPT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29547", str(script)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "SHARDLISTS-NCCL-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
