"""VecSimB200_LabelRangeQueryBatchDevice: device range batches answered per label, on multi-value indexes (DESIGN.md §4.12).

A label is in a query's answer iff one of its rows has score <= the radius (a NaN score never passes); its score is the smallest
such row score (brute_force_multi.h's unique_results_container).  Each batch takes the route of VecSimB200_RangeQueryBatchDevice;
a route's proven row answer is folded to labels by range_label_fold_kernel (one CTA per query, at most kRangeFoldMaxHits rows,
else flag 3 and the exact scan), and the exact scan folds label-major over the CSR label table (range_label_wide_kernel).

CPU: the reference's emplace sequence equals the fold rule; the route fold (sort by label, score key, row; first per label) and the
label-major fold give the same answer; the fold's constants are pinned to the sources.
GPU: every answer equals VecSimIndex_RangeQuery on the multi-value index per query (labels, float32 score bits, order, both
orders, count); negative inner-product radii are checked against the C restatement with multi=True.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle_lib as ol

_VT = {ol.F32: 0, ol.F16: 3, ol.BF16: 2, ol.I8: 4, ol.U8: 5}  # VecSimType
_MT = {ol.L2: 0, ol.IP: 1, ol.COS: 2}                          # VecSimMetric
BY_ID, BY_SCORE = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "redisearch_b200", "csrc")
FOLD_MAX_HITS = 4096  # kRangeFoldMaxHits (coarse_tc.h): hit rows the route fold sorts per query


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


def f32(x):
    return np.float32(x)


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


# ------------------------------------------------------------------------------------------------------------------
# CPU: the fold rule, restated
# ------------------------------------------------------------------------------------------------------------------
def _orderable_key(x):
    """orderable_key (topk_common.cuh): -0 -> +0, NaN -> the largest key"""
    x = f32(x)
    if np.isnan(x):
        return 0xFFFFFFFF
    u = int(np.array([x + f32(0.0)], dtype=np.float32).view(np.uint32)[0])
    return (~u) & 0xFFFFFFFF if u & 0x80000000 else u | 0x80000000


def _emplace(scores, labels, r):
    """brute_force.h rangeQuery with unique_results_container::emplace: rows in id order, score <= radius, first score of a
    label kept unless a later one is strictly smaller"""
    best = {}
    for s, lab in zip(scores, labels):
        if s <= r:
            if lab not in best:
                best[lab] = s
            elif best[lab] > s:
                best[lab] = s
    return best


def _route_fold(scores, labels, r):
    """range_label_fold_kernel: the hit rows sorted by (label, score key, row), the first of each label -> (key, row)"""
    hits = sorted((int(labels[i]), _orderable_key(scores[i]), i) for i in range(len(scores)) if scores[i] <= r)
    out = {}
    for lab, key, row in hits:
        if lab not in out:
            out[lab] = (key, row)
    return out


def _label_major_fold(scores, labels, r):
    """range_label_wide_kernel: per label, the smallest composite (key << 32 | row) over its rows with score <= r"""
    rows_of = {}
    for i, lab in enumerate(labels):
        rows_of.setdefault(int(lab), []).append(i)
    out = {}
    for lab, rows in rows_of.items():
        best = None
        for i in rows:
            if scores[i] <= r:
                c = (_orderable_key(scores[i]) << 32) | i
                best = c if best is None or c < best else best
        if best is not None:
            out[lab] = (best >> 32, best & 0xFFFFFFFF)
    return out


def _score_vectors(rng):
    for _ in range(300):
        n = int(rng.integers(1, 60))
        labels = rng.integers(0, max(1, n // 3), n)
        scores = f32(rng.integers(-4, 5, n)) * f32(0.25)  # ties
        scores[rng.random(n) < 0.15] = np.nan
        scores[rng.random(n) < 0.15] = f32(-0.0)
        scores[rng.random(n) < 0.1] = f32(0.0)
        for r in (f32(0.0), f32(-0.0), f32(0.25), f32(-0.5), f32(1.0), f32(np.inf), f32(np.nan)):
            yield scores, labels, r


def test_emplace_sequence_is_the_fold_rule():
    """min over the passing rows, the label absent if none passes; -0 and +0 are equal (the fold emits +0)"""
    for scores, labels, r in _score_vectors(np.random.default_rng(5)):
        want = _emplace(scores, labels, r)
        got = _route_fold(scores, labels, r)
        assert sorted(want) == sorted(int(x) for x in got), (scores, labels, r)
        for lab, (key, row) in got.items():
            assert key == _orderable_key(want[lab])
            assert f32(scores[row]) == want[lab] and scores[row] <= r
        if np.isnan(r):
            assert not got


def test_route_fold_equals_label_major_fold():
    for scores, labels, r in _score_vectors(np.random.default_rng(6)):
        assert _route_fold(scores, labels, r) == _label_major_fold(scores, labels, r)


def test_constants_match_the_sources():
    h, cu, host, api = _read("coarse_tc.h"), _read("coarse_tc.cu"), _read("vecsim_index.cpp"), \
        open(os.path.join(ROOT, "include", "vecsim_b200.h")).read()
    m = re.search(r"\bkRangeFoldMaxHits\s*=\s*(\d+)\s*;", h)
    assert m and int(m.group(1)) == FOLD_MAX_HITS
    assert "(size_t)kRangeFoldMaxHits * 12" in cu  # (label << 32 | key) + row per hit in shared memory: 48 KB
    # the dense label table's rule (-2): a label >= 2^32 - 1 or beyond 4 x rows + 2^24
    assert "if (max_label > 4 * count_ + (1u << 24) || max_label >= 0xFFFFFFFFull) return false;" in host
    assert "if (multi_ && !sync_label_table()) return -2;" in host
    assert "more than 4096" in api and "a label >= 2^32 - 1" in api


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mode1():
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    yield vs
    vs.lib().VecSimB200_SetCoarseMode(-1)


def scattered_labels(n, rng, lo=3, hi=5, first=1):
    """lo..hi rows per label, spread over the index; labels from `first`, spaced by 2 so label and row order differ"""
    c = rng.integers(lo, hi + 1, n)
    cs = np.cumsum(c)
    nl = int(np.searchsorted(cs, n)) + 1
    lab = np.repeat(first + 2 * np.arange(nl, dtype=np.uint64), c[:nl])[:n]
    return lab[rng.permutation(n)]


def _index(vtype, metric, dim, rows, labels, port=False, multi=True):
    vs = _vs()
    g = vs.VecSimIndex(_VT[vtype], dim, _MT[metric], multi=multi)
    assert g.add_many(rows, labels=labels) == len(rows)
    p = None
    if port:
        p = ol.PortIndex(vtype, dim, metric, multi=multi, tier=ol.TIER_AVX512)
        for r, lab in zip(rows, labels):
            p.add(r, int(lab))
    return g, p


def _stage(g, qs):
    import torch

    vs = _vs()
    nq = qs.shape[0]
    pitch = g.query_pitch()
    buf = np.zeros((nq, pitch), dtype=np.uint8)
    for i in range(nq):
        b = np.zeros(pitch, dtype=np.uint8)
        raw = np.ascontiguousarray(qs[i]).view(np.uint8)
        b[:raw.size] = raw
        if g.metric == _MT[ol.COS]:
            vs.normalize(b, g.dim, g.vtype)
        buf[i] = b
    return torch.from_numpy(buf).cuda()


def _run(g, qs, radii, cap, order, fn="label_range_batch_device"):
    import torch

    d_q = _stage(g, qs)
    d_r = torch.from_numpy(np.ascontiguousarray(radii, dtype=np.float32)).cuda()
    lab, sc, cnt, rc = getattr(g, fn)(d_q, d_r, cap, order)
    torch.cuda.synchronize()
    assert rc == 0
    return lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _flags(g, nq):
    f = np.zeros(nq, dtype=np.uint32)
    assert _vs().lib().VecSimB200_LastCoarseFlags(g.h, f.ctypes.data_as(C.c_void_p), nq) == 0
    return f


def _path(g):
    return _vs().lib().VecSimB200_LastBatchPath(g.h)


def _check(g, p, qs, radii, cap, order, lab, sc, cnt):
    for i in range(qs.shape[0]):
        r = float(radii[i])
        if r >= 0 or np.isnan(r):
            if np.isnan(r):
                ei, es = np.zeros(0, np.int64), np.zeros(0)
            else:
                ei, es, code = g.range(qs[i], r, order)
                assert code == 0
            ties = False
        else:  # the host API refuses a negative radius: the C restatement of the reference, multi=True
            ei, es = p.range(qs[i], r, order)
            ties = order == BY_SCORE
        n = len(ei)
        assert int(cnt[i]) == n, (i, r, int(cnt[i]), n)
        if n > cap:
            assert (lab[i] == -1).all() and np.isnan(sc[i]).all(), i
            continue
        gi, gs = lab[i, :n], sc[i, :n]
        if ties:
            a, b = np.lexsort((gi, gs)), np.lexsort((ei, es.astype(np.float32)))
            gi, gs, ei, es = gi[a], gs[a], ei[b], es[b]
        assert gi.tolist() == ei.tolist(), (i, r, gi[:8].tolist(), ei[:8].tolist(), n)
        assert gs.astype(np.float32).tobytes() == es.astype(np.float32).tobytes(), (i, r)
        assert (lab[i, n:] == -1).all() and np.isnan(sc[i, n:]).all(), i


def _radii_at(g, qs, ranks):
    """the ranks-th LABEL neighbour of each query (a multi-value KNN batch)"""
    labels, scores, rc = g.topk_batch(qs, max(ranks))
    assert rc == 0
    return np.array([scores[i, ranks[i % len(ranks)] - 1] for i in range(qs.shape[0])], dtype=np.float32)


# ------------------------------------------------------------------------------------------------------------------
# GPU: routes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim", [128, 768])
@pytest.mark.parametrize("metric", [ol.COS, ol.IP, ol.L2])
def test_fp32_route(mode1, metric, dim):
    n, nq = 70_000, 40
    rng = np.random.default_rng(dim + metric)
    rows = ol.synth_rows(ol.F32, 7, 0, n, dim)
    g, _ = _index(ol.F32, metric, dim, rows, scattered_labels(n, rng))
    qs = ol.synth_rows(ol.F32, 8, 0, nq, dim)
    if metric == ol.IP:
        qs = (qs.astype(np.float64) / dim).astype(np.float32)  # distances 1 - dot stay positive
    radii = _radii_at(g, qs, [1, 10, 100, 37])
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 128, order)
        assert _path(g) == 1 and _flags(g, nq).tolist() == [1] * nq
        _check(g, None, qs, radii, 128, order, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("metric", [ol.IP, ol.COS, ol.L2])
def test_8bit_route(mode1, vtype, metric):
    dim, n, nq = 128, 70_000, 32
    rng = np.random.default_rng(11 + metric)
    rows = ol.synth_rows(vtype, 11, 0, n, dim)
    labels = scattered_labels(n, rng)
    qs = ol.synth_rows(vtype, 12, 0, nq, dim)
    copies = [100, 20_000, 45_000, 69_999]
    rows[copies] = qs[0]  # one label whose rows are copies of query 0
    labels[copies] = 1_000_001
    g, p = _index(vtype, metric, dim, rows, labels, port=True)
    radii = _radii_at(g, qs, [10, 100])
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 256, order)
        assert _path(g) == 2 and _flags(g, nq).tolist() == [1] * nq, (_path(g), _flags(g, nq)[:8])
        _check(g, p, qs, radii, 256, order, lab, sc, cnt)
        assert 1_000_001 in lab[0, :int(cnt[0])].tolist()


@pytest.mark.gpu
def test_reference_scan(mode1):
    """a few queries against the reference's own multi-value range scan"""
    if ol.ref_vecsim() is None:
        pytest.skip("oracle/_ref is not built")
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(ol.I8, 21, 0, n, dim)
    labels = scattered_labels(n, np.random.default_rng(21))
    g, _ = _index(ol.I8, ol.L2, dim, rows, labels)
    ref = ol.RefIndex(ol.I8, dim, ol.L2, multi=True)
    for r, lab in zip(rows, labels):
        ref.add(r, int(lab))
    qs = ol.synth_rows(ol.I8, 22, 0, nq, dim)
    radii = _radii_at(g, qs, [10, 50])
    lab, sc, cnt = _run(g, qs, radii, 256, BY_ID)
    assert _path(g) == 2
    for i in range(4):
        ri, rs = ref.range(qs[i], float(radii[i]), BY_ID)
        assert int(cnt[i]) == len(ri)
        assert lab[i, :len(ri)].tolist() == ri.tolist()
        assert sc[i, :len(ri)].astype(np.float32).tobytes() == rs.astype(np.float32).tobytes()


@pytest.mark.gpu
def test_too_many_hit_rows_to_fold(mode1):
    """a proven query with more than kRangeFoldMaxHits hit rows spread so that no list overflows: flag 3, the exact scan's
    answer; the rest of the batch keeps flag 1"""
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(ol.I8, 31, 0, n, dim)
    labels = scattered_labels(n, np.random.default_rng(31))
    qs = ol.synth_rows(ol.I8, 32, 0, nq, dim)
    copies = np.arange(0, n, 14)[:5000]  # 5000 copies of query 0, one in 14 rows
    assert len(copies) > FOLD_MAX_HITS
    rows[copies] = qs[0]
    labels[copies] = 2_000_001 + 2 * (np.arange(len(copies)) // 2)  # 2500 labels of two copies each
    g, _ = _index(ol.I8, ol.L2, dim, rows, labels)
    radii = _radii_at(g, qs, [10])
    radii[0] = 0.0
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 4096, order)
        f = _flags(g, nq)
        assert _path(g) == 2 and f[0] == 3 and f[1:].tolist() == [1] * (nq - 1), f.tolist()
        assert int(cnt[0]) == 2500
        _check(g, None, qs, radii, 4096, order, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F32, ol.I8])
def test_chunked_labels_overflow_the_lists(mode1, vtype):
    """contiguous labels of near rows: a query among them overflows its lists, reports flag 0 and gets the exact label fold.
    fp32: labels of 200 rows, so that every 128-row tile of the query's own label holds more hits than a list (96) takes."""
    dim, n, nq = 128, 70_000, 16
    per = 200 if vtype == ol.F32 else 50
    rng = np.random.default_rng(41)
    labels = np.repeat(1 + np.arange(n // per, dtype=np.uint64), per)
    if vtype == ol.F32:
        centres = rng.standard_normal((n // per, dim)).astype(np.float32)
        rows = (np.repeat(centres, per, axis=0) + 0.05 * rng.standard_normal((n, dim))).astype(np.float32)
        qs = (centres[:nq] + 0.05 * rng.standard_normal((nq, dim))).astype(np.float32)
        ranks = [10]
    else:
        rows = ol.synth_rows(ol.I8, 41, 0, n, dim)
        base = rows[10].copy()
        base[0] = 50
        rows[20_000:60_000] = base  # 800 labels of near-duplicates
        rows[20_000:60_000, 0] = 50 + np.arange(40_000) % 3
        qs = ol.synth_rows(ol.I8, 42, 0, nq, dim)
        qs[3] = base
        ranks = [10]
    g, _ = _index(vtype, ol.L2, dim, rows, labels)
    radii = _radii_at(g, qs, ranks)
    if vtype == ol.I8:
        radii[3] = 400.0
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 1024, order)
        f = _flags(g, nq)
        assert _path(g) == (1 if vtype == ol.F32 else 2)
        if vtype == ol.F32:
            assert f.tolist() == [0] * nq, f.tolist()
        else:
            assert f[3] == 0 and int(cnt[3]) == 800, (f.tolist(), int(cnt[3]))
        _check(g, None, qs, radii, 1024, order, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["f16", "bf16", "mode0", "small", "nq15"])
def test_batches_off_the_routes(case):
    vs = _vs()
    vtype, metric, dim, n, nq = ol.F32, ol.L2, 64, 70_000, 16
    mode = 1
    if case in ("f16", "bf16"):
        vtype = ol.F16 if case == "f16" else ol.BF16
    elif case == "mode0":
        mode = 0
    elif case == "small":
        n = 20_000
    else:
        nq = 15
    vs.lib().VecSimB200_SetCoarseMode(mode)
    try:
        rows = ol.synth_rows(vtype, 61, 0, n, dim)
        g, _ = _index(vtype, metric, dim, rows, scattered_labels(n, np.random.default_rng(61)))
        qs = ol.synth_rows(vtype, 62, 0, nq, dim)
        radii = _radii_at(g, qs, [20])
        for order in (BY_SCORE, BY_ID):
            lab, sc, cnt = _run(g, qs, radii, 512, order)
            assert _path(g) == 0 and _flags(g, nq).tolist() == [0] * nq
            _check(g, None, qs, radii, 512, order, lab, sc, cnt)
    finally:
        vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: label edge cases
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_label_edges(mode1):
    """fp32 L2 on the fp32 route: a label with one row inside and one outside the radius; a label whose only passing row is
    its last; a radius exactly at a label's best row and one float below; a NaN radius; +inf with a small cap; cap equal to the
    label count while the rows exceed it, and one below"""
    dim, n, nq = 128, 70_000, 16
    rng = np.random.default_rng(71)
    rows = ol.synth_rows(ol.F32, 71, 0, n, dim)
    labels = scattered_labels(n, rng)
    q = ol.synth_rows(ol.F32, 72, 0, 1, dim)[0]
    A, B, Cl = 3_000_001, 3_000_003, 3_000_005

    def near(eps, j):
        r = q.copy()
        r[j % dim] += f32(eps)
        return r

    rows[1000], labels[1000] = near(0.01, 0), A   # A: one row inside ...
    labels[2000] = A                              # ... and one far row
    for j, pos in enumerate((3000, 3001, 3002)):  # B: three far rows, then its only passing row, added last
        labels[pos] = B
    rows[69_000], labels[69_000] = near(0.02, 1), B
    cpos = np.arange(5000, 65_000, 200)           # Cl: 300 near rows scattered
    for j, pos in enumerate(cpos):
        rows[pos], labels[pos] = near(0.03 + 1e-4 * j, j + 2), Cl
    g, _ = _index(ol.F32, ol.L2, dim, rows, labels)
    dA = g.range(q, 1e-3, BY_SCORE)[1][0]
    dA = f32(dA)
    d_far = f32(0.03 + 0.03 + 1e-4 * 300) ** 2
    qs = np.repeat(q[None], nq, axis=0)
    radii = np.array([dA, np.nextafter(dA, f32(-np.inf)), f32(0.02) ** 2 * f32(1.0001), np.nan, np.inf, d_far] + [dA] * 10,
                     dtype=np.float32)
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 16, order)
        _check(g, None, qs[:4], radii[:4], 16, order, lab, sc, cnt)
        assert lab[0, :int(cnt[0])].tolist() == [A] and int(cnt[1]) == 0
        assert sorted(lab[2, :int(cnt[2])].tolist()) == [A, B]
        assert int(cnt[3]) == 0 and (lab[3] == -1).all()
        assert int(cnt[4]) == len(np.unique(labels)) and (lab[4] == -1).all() and np.isnan(sc[4]).all()
        assert int(cnt[5]) == 3
    n_lab = 3  # radius d_far: A, B, Cl from 302 rows
    for cap, full in ((n_lab, True), (n_lab - 1, False)):
        for order in (BY_SCORE, BY_ID):
            lab, sc, cnt = _run(g, qs, radii, cap, order)
            assert int(cnt[5]) == n_lab
            if full:
                assert sorted(lab[5].tolist()) == [A, B, Cl]
                _check(g, None, qs[5:6], radii[5:6], cap, order, lab[5:6], sc[5:6], cnt[5:6])
            else:
                assert (lab[5] == -1).all() and np.isnan(sc[5]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F32, ol.I8])
def test_cosine_zero_row_beside_a_passing_row(mode1, vtype):
    """a zero row (NaN distance) never passes, its label is answered by its other row"""
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(vtype, 81, 0, n, dim)
    labels = scattered_labels(n, np.random.default_rng(81))
    qs = ol.synth_rows(vtype, 82, 0, nq, dim)
    rows[777] = 0
    rows[778] = qs[0]
    labels[777] = labels[778] = 4_000_001
    labels[779] = 4_000_003  # a label of one zero row
    rows[779] = 0
    g, p = _index(vtype, ol.COS, dim, rows, labels, port=True)
    radii = _radii_at(g, qs, [50])
    radii[1:4] = np.inf
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 4096, order)
        _check(g, p, qs, radii, 4096, order, lab, sc, cnt)
        assert 4_000_001 in lab[0, :int(cnt[0])].tolist()
        assert int(cnt[1]) == len(np.unique(labels)) - 1 and 4_000_003 not in lab[1, :int(cnt[1])].tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.F32])
def test_mutations_between_batches(mode1, vtype):
    """rows added to an existing label change its score, a deleted label disappears, swap-deletes move rows"""
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(vtype, 91, 0, n, dim)
    labels = scattered_labels(n, np.random.default_rng(91))
    g, _ = _index(vtype, ol.L2, dim, rows, labels)
    qs = ol.synth_rows(vtype, 92, 0, nq, dim)
    radii = _radii_at(g, qs, [10])
    _run(g, qs, radii, 256, BY_SCORE)
    grown = [int(labels[5_000 + 7 * i]) for i in range(nq)]
    for i in range(0, nq, 2):
        g.add(qs[i], grown[i])  # a copy of query i joins an existing label: its score becomes 0
    lab0, _, cnt0 = _run(g, qs, radii, 256, BY_SCORE)
    gone = [int(x) for x in lab0[1, :3]]
    for x in gone + [int(labels[0]), int(labels[n - 1])]:
        g.delete(x)
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 256, order)
        assert _path(g) == (2 if vtype == ol.I8 else 1)
        _check(g, None, qs, radii, 256, order, lab, sc, cnt)
        for i in range(0, nq, 2):
            got = lab[i, :int(cnt[i])].tolist()
            assert grown[i] in got and sc[i, got.index(grown[i])] == 0
        assert not set(gone) & set(lab[1, :int(cnt[1])].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F32, ol.I8])
def test_single_value_index_is_the_row_call(mode1, vtype):
    dim, n, nq = 128, 70_000, 32
    rows = ol.synth_rows(vtype, 101, 0, n, dim)
    g, _ = _index(vtype, ol.L2, dim, rows, np.arange(1, n + 1, dtype=np.uint64), multi=False)
    qs = ol.synth_rows(vtype, 102, 0, nq, dim)
    radii = _radii_at(g, qs, [10, 200])
    radii[3] = np.inf
    for order in (BY_SCORE, BY_ID):
        a = _run(g, qs, radii, 128, order)
        fa, pa = _flags(g, nq), _path(g)
        b = _run(g, qs, radii, 128, order, fn="range_batch_device")
        assert pa == _path(g) and fa.tolist() == _flags(g, nq).tolist()
        for x, y in zip(a, b):
            assert x.tobytes() == y.tobytes()


@pytest.mark.gpu
def test_outputs_feed_torch_on_the_callers_stream(mode1):
    import torch

    dim, n, nq = 128, 70_000, 64
    rows = ol.synth_rows(ol.I8, 111, 0, n, dim)
    g, _ = _index(ol.I8, ol.IP, dim, rows, scattered_labels(n, np.random.default_rng(111)))
    qs = ol.synth_rows(ol.I8, 112, 0, nq, dim)
    labels, scores, rc = g.topk_batch(qs, 10)
    radii = scores[:, 9].astype(np.float32)
    s = torch.cuda.Stream()
    d_q = _stage(g, qs)
    d_r = torch.from_numpy(radii).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        lab, sc, cnt, rc = g.label_range_batch_device(d_q, d_r, 64, BY_SCORE, stream=s)
        hits = (lab >= 0).sum(dim=1).to(torch.int32)  # consumed on the same stream, no host sync in between
        total = cnt.sum()
    s.synchronize()
    assert rc == 0
    assert hits.cpu().tolist() == cnt.cpu().tolist()
    assert int(total.item()) >= 10 * nq


@pytest.mark.gpu
def test_argument_checks(mode1):
    import torch

    vs = _vs()
    dim = 32
    rows = ol.synth_rows(ol.F32, 121, 0, 1000, dim)
    m = vs.VecSimIndex(0, dim, 0, multi=True)
    m.add_many(rows, labels=1 + np.arange(1000) // 3)
    qs = ol.synth_rows(ol.F32, 122, 0, 4, dim)
    d_q, d_r = _stage(m, qs), torch.ones(4, device="cuda")
    for cap, order in ((0, BY_SCORE), (4097, BY_SCORE), (16, 7)):
        out = torch.empty((4, max(cap, 1)), dtype=torch.int64, device="cuda")
        outs = torch.empty((4, max(cap, 1)), dtype=torch.float32, device="cuda")
        assert m.label_range_batch_device(d_q, d_r, cap, order, out_labels=out, out_scores=outs)[3] == -1
    assert m.label_range_batch_device(d_q[:0], d_r[:0], 16)[3] == 0
    assert m.label_range_batch_device(d_q, d_r, 16)[3] == 0
    for big in (2 ** 32 - 1, 2 ** 40, 4 * 1001 + 2 ** 24 + 5):
        s = vs.VecSimIndex(0, dim, 0, multi=True)
        s.add_many(rows, labels=1 + np.arange(1000) // 3)
        s.add(rows[0], big)
        lab = torch.full((4, 16), 7, dtype=torch.int64, device="cuda")
        sc = torch.full((4, 16), 3.0, dtype=torch.float32, device="cuda")
        cnt = torch.full((4,), 5, dtype=torch.int32, device="cuda")
        assert s.label_range_batch_device(d_q, d_r, 16, out_labels=lab, out_scores=sc, out_counts=cnt)[3] == -2, big
        torch.cuda.synchronize()
        assert (lab == 7).all() and (sc == 3.0).all() and (cnt == 5).all()
        s.close()
