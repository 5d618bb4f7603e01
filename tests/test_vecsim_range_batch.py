"""VecSimB200_RangeQueryBatch: nq range queries in one call.  Eligible fp32 batches take one fixed-bound main pass over the
fp16 shadow with the bound radius + eps per query, exact rescoring of the kept rows and a per-query proof (DESIGN.md §4,
"Range queries"); everything else is answered by the exact scan, query by query.  Either way every reply must be what
VecSimIndex_RangeQuery returns: the same ids in the same order with the same fp32 score bits as the reference (its compiled
code when oracle/_ref is built, else the C restatement at the AVX-512 tier) and as the per-query call on the same index.
"""
import math

import numpy as np
import pytest

import oracle_lib as ol
from test_coarse_adversarial import (EPS_F16, _checker, _metric_code, _normalized, _unit_query, adversarial_unit_rows, approx_dist,
                                     exact_dist, query_eps)


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


def _assert_reply(what, got, ref_ids, ref_scores, ties_any_order=False):
    """ties_any_order: rows of exactly equal score may come in any order among themselves (the reference sorts a range
    reply by score alone, so its order inside a run of ties is its sort's; this library orders them by label)."""
    ids, scores, code = got
    assert code == 0, (what, code)
    if ties_any_order:
        a, b = np.lexsort((ids, scores)), np.lexsort((ref_ids, ref_scores))
        ids, scores, ref_ids, ref_scores = ids[a], scores[a], ref_ids[b], ref_scores[b]
    assert ids.tolist() == ref_ids.tolist(), (what, ids[:12].tolist(), ref_ids[:12].tolist(), len(ids), len(ref_ids))
    assert scores.astype(np.float32).tobytes() == ref_scores.astype(np.float32).tobytes(), what


def _check_batch(g, p, qs, radii, order, replies, ref_every=1):
    """Every reply against VecSimIndex_RangeQuery on the same index (ids, order and score bits); every ref_every-th also
    against the reference (BY_SCORE: the order inside a run of exactly tied scores aside)."""
    for i in range(qs.shape[0]):
        gi, gs, gc = g.range(qs[i], float(radii[i]), order)
        _assert_reply((i, "per-query call"), replies[i], gi, gs)
        if i % ref_every == 0:
            pi, ps = p.range(qs[i], float(radii[i]), order)
            _assert_reply((i, "reference"), replies[i], pi, ps, ties_any_order=order == 0)


def _radii_at(g, qs, ranks):
    """Per query the exact distance of its ranks[i]-th neighbour (1-based; 0 = just below the nearest), from one exact
    top-100 batch (bit-equal to the reference: test_vecsim_coarse)."""
    labels, scores, rc = g.topk_batch(qs, 100)
    assert rc == 0
    d = scores.astype(np.float32)
    out = np.empty(qs.shape[0], dtype=np.float64)
    for i, r in enumerate(ranks):
        if r == 0:
            assert d[i, 0] > 0
            out[i] = float(np.nextafter(d[i, 0], np.float32(-np.inf)))
        else:
            out[i] = float(d[i, r - 1])
    return out


def _queries(metric, seed, nq, dim):
    qs = ol.synth_rows(ol.F32, seed, 0, nq, dim)
    if metric == ol.IP:  # raw inner product: distances 1 - dot stay positive (a radius must be >= 0)
        qs = (qs.astype(np.float64) / dim).astype(np.float32)
    return qs


# ------------------------------------------------------------------------------------------------------------------
# CPU: the worst-case rounding construction keeps its power at the radius
# ------------------------------------------------------------------------------------------------------------------
def _planted(metric, q_unit, scale, nb):
    """Row A and nb rows B around the unit query (adversarial_unit_rows), in the form the index stores them and the
    query as the caller passes it.  Raw inner product / L2: the rows scaled by `scale` (a power of two keeps their
    fp16 rounding); L2 scales the query likewise, inner product scales it by 1 / (2 scale), so that A's distance
    1 - dot stays positive (a radius must be >= 0)."""
    a, b = adversarial_unit_rows(q_unit, nb)
    if metric == ol.COS:
        return _normalized(a), _normalized(b), q_unit
    sa = (a.astype(np.float64) * scale).astype(np.float32)
    sb = (b.astype(np.float64) * scale).astype(np.float32)
    qf = scale if metric == ol.L2 else 1.0 / (2.0 * scale)
    return sa, sb, (q_unit.astype(np.float64) * qf).astype(np.float32)


def _eps(metric, max_norm, q, dim):
    if metric == ol.COS:
        return EPS_F16
    return query_eps(EPS_F16, max_norm, float(np.linalg.norm(q.astype(np.float64))), dim, metric == ol.L2)


@pytest.mark.parametrize("dim", [128, 768])
@pytest.mark.parametrize("metric", [ol.COS, ol.IP, ol.L2])
def test_rounding_builder_has_power_at_the_radius(metric, dim):
    """Radius = A's exact distance.  A's approximate distance lies at least eps / 4 above it (so a bound of radius + eps / 4
    drops A), and some B rows lie at or below it in approximate distance while their exact distance is above (so only the
    exact rescoring keeps them out)."""
    rng = np.random.default_rng(dim + metric)
    scale = 16.0
    for _ in range(4):
        q = _normalized(_unit_query(rng, dim))
        sa, sb, qq = _planted(metric, q, scale, 11)
        mx = float(np.sqrt(max((sa.astype(np.float64) ** 2).sum(), (sb.astype(np.float64) ** 2).sum(1).max())))
        e = _eps(metric, mx, qq, dim)
        r = float(np.float32(exact_dist(sa, qq, metric)))
        assert r > 0
        pa, pb, eb = approx_dist(sa, qq, metric), approx_dist(sb, qq, metric), exact_dist(sb, qq, metric)
        assert pa - r >= e / 4, (pa - r, e)
        assert pa - r < e  # ... and the proof's bound still reaches it
        assert ((pb <= r) & (eb > r)).any()


# ------------------------------------------------------------------------------------------------------------------
# GPU: parity matrix
# ------------------------------------------------------------------------------------------------------------------
# every metric, dim, corpus size and batch size appears; each batch mixes the four radius kinds and is run in both orders
_MATRIX = [
    (ol.COS, 32, 70_000, 16), (ol.COS, 128, 300_000, 256), (ol.COS, 768, 70_000, 40), (ol.COS, 1016, 70_000, 16),
    (ol.IP, 32, 300_000, 40), (ol.IP, 128, 70_000, 16), (ol.IP, 768, 70_000, 256), (ol.IP, 1016, 70_000, 40),
    (ol.L2, 32, 70_000, 256), (ol.L2, 128, 70_000, 40), (ol.L2, 768, 300_000, 16), (ol.L2, 1016, 70_000, 16),
]


@pytest.mark.gpu
@pytest.mark.parametrize("metric,dim,n,nq", _MATRIX)
def test_range_batch_parity(metric, dim, n, nq):
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    rows = ol.synth_rows(ol.F32, 201, 0, n, dim)
    qs = _queries(metric, 202, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    ranks = [(1, 10, 100, 0)[i % 4] for i in range(nq)]
    radii = _radii_at(g, qs, ranks)
    for order in (vs.BY_SCORE, vs.BY_ID):
        replies, rc, flags = g.range_batch(qs, radii, order)
        assert rc == 0
        _check_batch(g, p, qs, radii, order, replies, ref_every=1 if order == vs.BY_SCORE else 4)
        hit = np.array([r > 0 for r in ranks])
        assert (flags[hit] == 1).sum() >= 0.9 * hit.sum(), flags.tolist()
        for i, r in enumerate(ranks):
            if r == 0:
                assert len(replies[i][0]) == 0
            else:
                assert len(replies[i][0]) >= r
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
def test_radius_is_inclusive():
    """A radius equal to a row's reference distance returns that row; the next float below it does not."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq = 70_000, 128, 16
    rows = ol.synth_rows(ol.F32, 211, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 212, 0, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    pl, ps = zip(*(p.topk(qs[i], 10) for i in range(nq)))
    at = np.array([float(s[9]) for s in ps])
    replies, rc, flags = g.range_batch(qs, at)
    assert rc == 0 and (flags == 1).all(), flags.tolist()
    for i in range(nq):
        assert int(pl[i][9]) in replies[i][0].tolist()
    below = np.array([float(np.nextafter(np.float32(x), np.float32(-np.inf))) for x in at])
    replies, rc, flags = g.range_batch(qs, below)
    assert rc == 0 and (flags == 1).all()
    for i in range(nq):
        assert int(pl[i][9]) not in replies[i][0].tolist() or float(ps[i][8]) == float(ps[i][9])
    _check_batch(g, p, qs, below, vs.BY_SCORE, replies)
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [128, 768])
@pytest.mark.parametrize("metric", [ol.COS, ol.IP, ol.L2])
def test_worst_case_rounding_at_the_radius(metric, dim):
    """Per query: row A at exactly the radius, rounded by the fp16 operands to 0.3-0.4 eps above it, and rows B rounded
    below the radius although their exact distance is above it.  The batch must return A and no B, proven: a bound
    without eps (or with eps / 4) drops A, and keeping rows by their approximate distance admits the B rows."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    n, nq, nb = 70_000, 16, 11
    rng = np.random.default_rng(3000 + dim + metric)
    rows = ol.synth_rows(ol.F32, 221, 0, n, dim)
    scale = 1.0 if metric == ol.COS else 2.0 ** math.ceil(math.log2(float(np.sqrt((rows.astype(np.float64) ** 2).sum(1).max()))))
    pos = rng.permutation(n)[: nq * (nb + 1)].reshape(nq, nb + 1)  # spread over the row ranges: no list overflows
    qs = np.empty((nq, dim), dtype=np.float32)
    for i in range(nq):
        q = _normalized(_unit_query(rng, dim))
        sa, sb, qs[i] = _planted(metric, q, scale, nb)
        rows[pos[i, 0]] = sa
        rows[pos[i, 1:]] = sb
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    radii = np.empty(nq)
    for i in range(nq):  # A is the nearest row: its reference distance
        pi, ps = p.topk(qs[i], 1)
        assert int(pi[0]) == pos[i, 0] + 1
        radii[i] = float(ps[0])
    replies, rc, flags = g.range_batch(qs, radii)
    assert rc == 0
    _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    max_norm = float(np.sqrt(np.max((rows.astype(np.float64) ** 2).sum(1))))
    for i in range(nq):
        ids = replies[i][0].tolist()
        assert pos[i, 0] + 1 in ids and not set((pos[i, 1:] + 1).tolist()) & set(ids), i
        # the construction has power on the rows the index actually stores
        st = np.empty((nb + 1, dim), dtype=np.float32)
        for j, r in enumerate(pos[i]):
            assert g.L.VecSimB200_ReadRows(g.h, int(r), 1, st[j].ctypes.data) == 0
        e = _eps(metric, max_norm, qs[i], dim)
        r = radii[i]
        assert approx_dist(st[0], qs[i], metric) - r >= e / 4
        pb, eb = approx_dist(st[1:], qs[i], metric), exact_dist(st[1:], qs[i], metric)
        assert ((pb <= r) & (eb > r)).any()
    assert (flags == 1).all(), flags.tolist()
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
def test_overflowing_queries_fall_back_and_the_rest_stay_on_the_route():
    """Query 0 has a radius of +inf (every row), query 1 sits on a cluster of 120 near-duplicates inside one row tile (more
    rows of one row range within the bound than its 96-slot list holds).  Both are answered by the exact scan (flag 0)
    with the reference's answer; the other queries of the batch stay proven."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq = 70_000, 128, 24
    rng = np.random.default_rng(231)
    rows = ol.synth_rows(ol.F32, 231, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 232, 0, nq, dim)
    center = rng.uniform(-1, 1, dim)
    rows[5 * 128: 5 * 128 + 120] = (center[None, :] + 1e-3 * rng.standard_normal((120, dim))).astype(np.float32)
    qs[1] = center.astype(np.float32)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    radii = _radii_at(g, qs, [10] * nq)
    radii[0] = math.inf
    radii[1] = 1e-3  # the whole cluster (cosine distance ~1e-6 .. 1e-5), nothing else
    replies, rc, flags = g.range_batch(qs, radii)
    assert rc == 0
    _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    assert len(replies[0][0]) == n and len(replies[1][0]) == 120
    assert flags[0] == 0 and flags[1] == 0 and (flags[2:] == 1).all(), flags.tolist()
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.L2])
def test_edge_inputs(metric):
    """NaN radius: empty reply, as in the reference.  Raw queries with a component of 65520 or 1e5 (not finite in fp16):
    answered exactly, flag 0.  Negative radius and invalid order: -1, no replies."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq = 70_000, 64, 16
    rows = ol.synth_rows(ol.F32, 241, 0, n, dim)
    qs = _queries(metric, 242, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs[1, 0], qs[2, 0] = np.float32(65520.0), np.float32(1e5)
    radii = _radii_at(g, qs, [10] * nq)
    radii[0] = math.nan
    if metric == ol.IP:  # the nearest distances of the two are far below 0: take the rows with dot >= 0.5 instead
        radii[1] = radii[2] = 0.5
    replies, rc, flags = g.range_batch(qs, radii)
    assert rc == 0
    _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    assert len(replies[0][0]) == 0 and p.range(qs[0], math.nan)[0].size == 0
    assert len(replies[1][0]) > 0 and len(replies[2][0]) > 0
    assert (flags[:3] == 0).all() and (flags[3:] == 1).all(), flags.tolist()
    g.topk(qs[3], 1)
    assert g.debug_info()["LAST_SEARCH_MODE"] == "STANDARD_KNN"
    assert g.range_batch(qs[3:], radii[3:])[1] == 0
    assert g.debug_info()["LAST_SEARCH_MODE"] == "RANGE_QUERY"
    for bad_radii, order in ((np.where(np.arange(nq) == 5, -0.5, radii), vs.BY_SCORE), (radii, 7)):
        reps, rc, flags = g.range_batch(qs, bad_radii, order)
        assert rc == -1 and reps == []
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: batches that take the exact scan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["multi", "f16", "int8", "mode0", "mode2", "small"])
def test_exact_path(case):
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode({"mode0": 0, "mode2": 2}.get(case, 1))
    n, dim, nq = (60_000 if case == "small" else 70_000), 128, 16
    vtype = {"f16": ol.F16, "int8": ol.I8}.get(case, ol.F32)
    vcode = {ol.F32: vs.VecSimType_FLOAT32, ol.F16: vs.VecSimType_FLOAT16, ol.I8: vs.VecSimType_INT8}[vtype]
    g = vs.VecSimIndex(vcode, dim, vs.VecSimMetric_Cosine, multi=case == "multi")
    rows = ol.to_type(ol.synth_rows(ol.F32, 251, 0, n, dim), vtype) if vtype != ol.F32 else ol.synth_rows(ol.F32, 251, 0, n, dim)
    if case == "multi":  # two vectors per label
        for lab in range(n // 2):
            g.add(rows[2 * lab], lab + 1)
            g.add(rows[2 * lab + 1], lab + 1)
    else:
        assert g.add_many(rows, label0=1) == n
    qs = ol.to_type(ol.synth_rows(ol.F32, 252, 0, nq, dim), vtype) if vtype != ol.F32 else ol.synth_rows(ol.F32, 252, 0, nq, dim)
    radii = np.array([float(g.topk(qs[i], 10)[1][-1]) for i in range(nq)])
    for order in (vs.BY_SCORE, vs.BY_ID):
        replies, rc, flags = g.range_batch(qs, radii, order)
        assert rc == 0 and (flags == 0).all()
        for i in range(nq):
            gi, gs, _ = g.range(qs[i], float(radii[i]), order)
            _assert_reply(i, replies[i], gi, gs)
            assert len(gi) >= 10 or case == "multi"
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: updates and timeouts
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.COS, ol.L2])
def test_updates_between_batches(metric):
    """Appends, raw overwrites and deletes between two batches are reflected in the second."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq = 70_000, 128, 16
    rows = ol.synth_rows(ol.F32, 261, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 262, 0, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    radii = _radii_at(g, qs, [10] * nq)
    replies, rc, flags = g.range_batch(qs, radii)
    assert rc == 0 and (flags == 1).sum() >= 0.9 * nq
    _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    # the nearest row of query 0 goes, query 1 gets a new row on top of it, label 5 is overwritten with query 2, label
    # 7 (and a far row) are deleted
    first0 = int(replies[0][0][0])
    assert g.delete(first0) == 1 and p.delete(first0) == 1
    new = (qs[1].astype(np.float64) + 1e-4).astype(np.float32)
    assert g.add(new, n + 1) == 1
    p.add(new, n + 1)
    assert g.add(qs[2], 5) == 0
    p.add(qs[2], 5)
    for lab in (7, n // 2):
        assert g.delete(lab) == 1 and p.delete(lab) == 1
    replies, rc, flags = g.range_batch(qs, radii)
    assert rc == 0
    _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    assert first0 not in replies[0][0].tolist() and n + 1 in replies[1][0].tolist() and 5 in replies[2][0].tolist()
    vs.lib().VecSimB200_SetCoarseMode(-1)


_KEEPALIVE = []


@pytest.mark.gpu
def test_timeout_marks_every_reply_and_the_next_call_succeeds():
    vs = _vs()
    L = vs.lib()
    L.VecSimB200_SetCoarseMode(1)
    n, dim, nq = 300_000, 128, 32
    rows = ol.synth_rows(ol.F32, 271, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 272, 0, nq, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    radii = _radii_at(g, qs, [10] * nq)
    calls = [0]

    def fire_after_first(ctx):  # passes the check on entry, fires while the pass runs (or right after)
        calls[0] += 1
        return 1 if calls[0] > 1 else 0

    cb, cb_off = vs.TIMEOUT_CB(fire_after_first), vs.TIMEOUT_CB(lambda ctx: 0)
    _KEEPALIVE.extend([cb, cb_off])
    try:
        for fire in (cb, vs.TIMEOUT_CB(lambda ctx: 1)):
            _KEEPALIVE.append(fire)
            calls[0] = 0
            L.VecSim_SetTimeoutCallbackFunction(fire)
            replies, rc, flags = g.range_batch(qs, radii)
            assert rc == vs.VecSim_QueryReply_TimedOut
            assert all(code == vs.VecSim_QueryReply_TimedOut for _, _, code in replies)
        L.VecSim_SetTimeoutCallbackFunction(cb_off)
        replies, rc, flags = g.range_batch(qs, radii)
        assert rc == 0 and (flags == 1).sum() >= 0.9 * nq
        _check_batch(g, p, qs, radii, vs.BY_SCORE, replies)
    finally:
        L.VecSim_SetTimeoutCallbackFunction(cb_off)
        L.VecSimB200_SetCoarseMode(-1)
