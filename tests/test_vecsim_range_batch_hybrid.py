"""VecSimB200_HybridRangeQueryBatchDevice: filtered range batches on the device (DESIGN.md §4.13).

Query i's answer is VecSimB200_LabelRangeQueryBatchDevice's answer for (query i, radius i) restricted to the docIds of filter i:
the same labels, score bits, order and counts.  A batch takes the range form of the ragged gather, or (single-value fp32 / int8 /
uint8 batches the range routes serve) the fixed-bound or fixed-radius pass with the filter bitmaps applied, the gather answering
what that pass leaves open.

CPU: the mode choice and the route eligibility restated and pinned to the sources; a numpy model of the multi-value range fold
next to getDistanceFrom's fold, with a NaN row first, in the middle and last.
GPU: every row equals LabelRangeQueryBatchDevice (cap 4096) restricted to the filter, bit for bit, across types, metrics,
multi-value indexes, orders, policies, filters, radii, caps, list overflow, pending posting-list filters, mutations and stream
order; 8 queries are checked against the reference's distances over rows read back from HBM.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "redisearch_b200", "csrc")
_VT = {ol.F32: 0, ol.F16: 3, ol.BF16: 2, ol.I8: 4, ol.U8: 5}  # VecSimType
_MT = {ol.L2: 0, ol.IP: 1, ol.COS: 2}                          # VecSimMetric
BY_SCORE, BY_ID = 0, 1  # VecSimQueryReply_Order
EMPTY_MODE, HYBRID_ADHOC_BF, HYBRID_BATCHES = 0, 2, 3
MIN_DENSE = 16  # kHybridRangeMinDense (vecsim_index.cpp)
F32_BYTES = {ol.F32: 4, ol.F16: 2, ol.BF16: 2, ol.I8: 1, ol.U8: 1}


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


# ------------------------------------------------------------------------------------------------------------------
# CPU: the mode choice
# ------------------------------------------------------------------------------------------------------------------
def dense_pays(caps, stored_bytes, pass_bytes, n):
    """hybrid_range_dense_pays: the gathers' bytes against the main pass's rows, two passes over a bitmap per query, the lists"""
    cap_sum = float(sum(caps))
    gather = cap_sum * (stored_bytes + 8)
    bitmaps = len(caps) * ((n + 31) // 32) * 4 * 2
    return gather > pass_bytes + bitmaps + 8.0 * cap_sum


def route(vtype, multi, n, dim, caps, policy=EMPTY_MODE, shadow=False):
    """The batch's route: 1 fp32 dense, 2 8-bit dense, 0 gather (coarse mode 1, fixed bound on, supported dims)."""
    if policy == HYBRID_ADHOC_BF or multi or n < 65536:
        return 0
    nq = len(caps)
    r8 = vtype in (ol.I8, ol.U8) and nq >= MIN_DENSE
    r32 = vtype == ol.F32 and (nq >= MIN_DENSE or shadow)
    if not (r8 or r32):
        return 0
    stored = dim * F32_BYTES[vtype]
    pass_bytes = n * dim * (1 if r8 else 2)
    if policy == HYBRID_BATCHES or dense_pays(caps, stored, pass_bytes, n):
        return 2 if r8 else 1
    return 0


def test_mode_choice_constants_are_the_sources():
    src = _read("vecsim_index.cpp")
    assert re.search(r"kHybridRangeMinDense = %d;" % MIN_DENSE, src)
    body = src[src.index("static bool hybrid_range_dense_pays"):]
    body = body[: body.index("\n}\n")]
    assert "(double)cap_sum * (double)(stored_bytes + 8)" in body
    assert "(double)nq * ((n + 31) / 32) * 4 * 2" in body
    assert "gather > pass_bytes + bitmaps + 8.0 * (double)cap_sum" in body
    fn = src[src.index("int FlatIndex::hybrid_range_batch_device"):]
    fn = fn[: fn.index("\n}\n")]
    assert "(double)n * dim_ * (r8 ? 1 : 2)" in fn  # the 8-bit rows, or the fp16 shadow
    assert "!multi_" in fn and "policy != HYBRID_ADHOC_BF" in fn
    assert "nq >= kHybridRangeMinDense || single_query_takes_coarse(1)" in fn


def test_mode_choice_puts_the_benchmark_on_both_sides():
    """10M x 768: 0.1 % filters stay on the gather, 10 % at 256 queries go dense, for fp32 and int8."""
    n, dim = 10_000_000, 768
    for vtype in (ol.F32, ol.I8):
        for nq in (16, 256):
            assert route(vtype, False, n, dim, [n // 1000] * nq) == 0
        assert route(vtype, False, n, dim, [n // 10] * 256) == (1 if vtype == ol.F32 else 2)
        assert route(vtype, False, n, dim, [n // 2] * 16) == (1 if vtype == ol.F32 else 2)
        # forced policies, and what is never eligible
        assert route(vtype, False, n, dim, [10] * 16, HYBRID_BATCHES) != 0
        assert route(vtype, False, n, dim, [n] * 16, HYBRID_ADHOC_BF) == 0
        assert route(vtype, True, n, dim, [n] * 16, HYBRID_BATCHES) == 0
    for vtype in (ol.F16, ol.BF16):
        assert route(vtype, False, n, dim, [n] * 256, HYBRID_BATCHES) == 0
    # below 16 queries: fp32 only once the shadow exists, 8-bit never
    assert route(ol.F32, False, n, dim, [n] * 15) == 0 and route(ol.F32, False, n, dim, [n] * 15, shadow=True) == 1
    assert route(ol.I8, False, n, dim, [n] * 15, HYBRID_BATCHES) == 0


def test_no_cap_floor_the_whole_batch_decides():
    """One broad filter can carry a batch of narrow ones: the rule sums the caps, there is no per-query floor."""
    n, dim = 1_000_000, 128
    narrow = [100] * 31
    assert route(ol.F32, False, n, dim, narrow + [100]) == 0
    assert route(ol.F32, False, n, dim, narrow + [n]) == 1


# ------------------------------------------------------------------------------------------------------------------
# CPU: the multi-value range fold
# ------------------------------------------------------------------------------------------------------------------
def get_distance_fold(ds):
    """gather_min_kernel / getDistanceFrom_Unsafe: dist = +inf, then dist = (dist < d) ? dist : d row by row"""
    dist = np.float32(np.inf)
    for d in ds:
        dist = dist if dist < d else np.float32(d)
    return dist


def range_fold(ds, r):
    """the range form: the smallest row score among the rows with score <= r (None when no row passes)"""
    passing = [np.float32(d) for d in ds if d <= r]
    return min(passing) if passing else None


@pytest.mark.parametrize("pos", ["first", "middle", "last"])
def test_range_fold_skips_nan_rows_where_the_distance_fold_does_not(pos):
    rows = [np.float32(0.1), np.float32(0.5)]
    nan = np.float32(np.nan)
    ds = {"first": [nan] + rows, "middle": [rows[0], nan, rows[1]], "last": rows + [nan]}[pos]
    r = np.float32(1.0)
    assert range_fold(ds, r) == np.float32(0.1)
    g = get_distance_fold(ds)
    if pos == "first":
        assert g == np.float32(0.1)  # NaN replaced by the next row
    elif pos == "middle":
        assert g == np.float32(0.5)  # the NaN reset the fold: 0.1 is lost
    else:
        assert np.isnan(g)  # the label would be dropped
    assert range_fold(ds, np.float32(0.3)) == np.float32(0.1)
    assert range_fold(ds, np.float32(0.05)) is None
    assert range_fold(ds, nan) is None


def test_range_fold_equals_the_label_answer_rule():
    """Without NaN rows the range fold keeps a label iff its getDistanceFrom distance is <= r, at that distance."""
    rng = np.random.default_rng(3)
    for _ in range(2000):
        ds = rng.random(rng.integers(1, 6)).astype(np.float32)
        r = np.float32(rng.random())
        f = range_fold(ds, r)
        g = get_distance_fold(ds)
        assert (f is not None) == (g <= r) and (f is None or f == g)


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


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stage(g, qs):
    """stored-form queries, query_pitch() apart, as a CUDA tensor"""
    vs = _vs()
    pitch = g.query_pitch()
    buf = np.zeros((len(qs), pitch), dtype=np.uint8)
    for i in range(len(qs)):
        b = np.zeros(pitch, dtype=np.uint8)
        raw = np.ascontiguousarray(qs[i]).view(np.uint8)
        b[: raw.size] = raw
        if g.metric == _MT[ol.COS]:
            vs.normalize(b, g.dim, g.vtype)
        buf[i] = b
    return _dev(buf)


def _params(policy):
    if policy is None:
        return None
    p = _vs().VecSimQueryParams()
    p.searchMode = policy
    return p


class Filters:
    """Device buffers of ascending filters: caps (default the sizes) may exceed the counts, the buffers then hold ids past the
    count that must never be read; exact_caps: no count pointers."""

    def __init__(self, filters, caps=None, exact_caps=False):
        self.filters = filters
        self.bufs, self.cnts, self.ptrs, self.caps, self.cptrs = [], [], [], [], []
        for i, f in enumerate(filters):
            cap = len(f) if caps is None else caps[i]
            buf = np.full(max(cap, 1), 0xFFFFFFF0, dtype=np.uint32)
            buf[: len(f)] = f
            self.bufs.append(_dev(buf.view(np.int32)))
            self.cnts.append(_dev(np.array([len(f)], dtype=np.int32)))
            self.ptrs.append(self.bufs[-1].data_ptr() if cap else None)
            self.cptrs.append(self.cnts[-1].data_ptr())
            self.caps.append(cap)
        if exact_caps:
            self.cptrs = None


def _flags(g, nq):
    f = np.zeros(nq, dtype=np.uint32)
    assert _vs().lib().VecSimB200_LastCoarseFlags(g.h, f.ctypes.data_as(C.c_void_p), nq) == 0
    return f


def _path(g):
    return _vs().lib().VecSimB200_LastBatchPath(g.h)


def hybrid(g, qd, rd, cap, fl, order=BY_SCORE, policy=None, stream=None):
    import torch

    lab, sc, cnt, modes, rc = g.hybrid_range_batch_device(qd, rd, cap, fl.ptrs, fl.caps, counts=fl.cptrs, order=order,
                                                          params=_params(policy), stream=stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32).astype(np.int64), modes, _flags(g, len(fl.caps))


def want(g, qd, rd, filters, order):
    """LabelRangeQueryBatchDevice at cap 4096, restricted to each filter (None where the whole answer exceeds 4096)"""
    import torch

    lab, sc, cnt, rc = g.label_range_batch_device(qd, rd, 4096, order)
    torch.cuda.synchronize()
    assert rc == 0
    lab, sc, cnt = lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
    out = []
    for i, f in enumerate(filters):
        c = int(cnt[i])
        if c > 4096:
            out.append(None)
            continue
        m = np.isin(lab[i, :c], np.asarray(f, dtype=np.int64))
        out.append((lab[i, :c][m], sc[i, :c][m]))
    return out


def check_rows(got, exp, cap, skip_unknown=False):
    lab, sc, cnt = got[:3]
    checked = 0
    for i, e in enumerate(exp):
        if e is None:
            assert skip_unknown, i
            continue
        n = len(e[0])
        assert cnt[i] == n, (i, int(cnt[i]), n)
        if n > cap:
            assert (lab[i] == -1).all() and np.isnan(sc[i]).all(), i
        else:
            assert lab[i, :n].tolist() == e[0].tolist(), (i, lab[i, :8].tolist(), e[0][:8].tolist())
            assert sc[i, :n].tobytes() == e[1].tobytes(), i
            assert (lab[i, n:] == -1).all() and np.isnan(sc[i, n:]).all(), i
        checked += 1
    return checked


def _index(vtype, metric, n, dim, multi=False, seed=42, deletes=True):
    """docIds 1..n (multi-value: 2 rows per docId); with `deletes`, 200 swap-deletes so docIds no longer follow rows"""
    vs = _vs()
    g = vs.VecSimIndex(_VT[vtype], dim, _MT[metric], multi=multi)
    rows = ol.synth_rows(vtype, seed, 0, n, dim)
    if multi:
        assert g.add_many(rows, labels=(np.arange(n, dtype=np.uint64) // 2 + 1)) == n
    else:
        assert g.add_many(rows, label0=1) == n
    deleted = []
    if deletes:
        top = n // 2 if multi else n
        deleted = list(range(1, top, top // 200))[:200]
        for d in deleted:
            assert g.delete(d) >= 1
    return g, deleted


def _filters(rng, top, nq, deleted, fracs):
    """ascending filters over docIds 1..top + 100 (the tail absent), cycling through the fractions; 'lt10' = fewer than 10
    entries; every filter but the empty one holds a few deleted docIds"""
    out = []
    for i in range(nq):
        fr = fracs[i % len(fracs)]
        if fr == "empty":
            out.append(np.zeros(0, np.uint32))
            continue
        m = 7 if fr == "lt10" else min(top + 100, max(1, int(fr * top)))
        f = set(rng.choice(np.arange(1, top + 101), m, replace=False).tolist()) | set(deleted[i % 7 :: 37])
        out.append(np.array(sorted(f), dtype=np.uint32))
    return out


FRACS = ["empty", "lt10", 0.001, 0.01, 0.1, 0.5, 1.0]


def _radii(g, qs, fl, ranks=(1, 10, 100, 1000)):
    """Per query: the whole corpus's ranks[i]-th distance, or (every third query) the 10th distance within its filter when that
    is smaller (a radius at a filtered neighbour)"""
    import torch

    kmax = max(ranks)
    labels, scores, rc = g.topk_batch(qs, kmax)
    assert rc == 0
    r = np.array([scores[i, ranks[i % len(ranks)] - 1] for i in range(len(qs))], dtype=np.float32)
    qd = _stage(g, qs)
    lab, sc, cnt, rc2 = g.topk_filtered_batch_device(qd, 10, fl.ptrs, fl.caps, counts=fl.cptrs)
    assert rc2 == 0
    torch.cuda.synchronize()
    sc, cnt = sc.cpu().numpy(), cnt.cpu().numpy()
    for i in range(0, len(qs), 3):
        if cnt[i] > 0:
            r[i] = min(r[i], sc[i, cnt[i] - 1])
    r[np.isnan(r)] = np.float32(0.5)
    return r


VARIANTS = [(ol.F32, ol.COS, False), (ol.F32, ol.L2, False), (ol.F32, ol.IP, False),
            (ol.I8, ol.L2, False), (ol.I8, ol.IP, False), (ol.I8, ol.COS, False),
            (ol.U8, ol.L2, False), (ol.U8, ol.IP, False), (ol.U8, ol.COS, False),
            (ol.F16, ol.IP, False), (ol.BF16, ol.L2, False),
            (ol.F32, ol.COS, True), (ol.F16, ol.L2, True), (ol.BF16, ol.IP, True), (ol.I8, ol.L2, True), (ol.U8, ol.COS, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,multi", VARIANTS)
def test_rows_equal_the_label_range_batch_restricted(mode1, vtype, metric, multi):
    rng = np.random.default_rng(hash((vtype, metric, multi)) % 1000)
    n, dim, nq = 70_000, 128, 32
    g, deleted = _index(vtype, metric, n, dim, multi=multi)
    top = n // 2 if multi else n
    qs = ol.synth_rows(vtype, 7, 0, nq, dim)
    filters = _filters(rng, top, nq, deleted, FRACS)
    fl = Filters(filters)
    radii = _radii(g, qs, fl, ranks=(1, 10, 100) if multi else (1, 10, 100, 1000))  # multi-value batches: k <= 128
    qd, rd = _stage(g, qs), _dev(radii)
    dense = 0 if multi or vtype in (ol.F16, ol.BF16) else (1 if vtype == ol.F32 else 2)
    for order in (BY_SCORE, BY_ID):
        exp = want(g, qd, rd, filters, order)
        for policy in (None, HYBRID_ADHOC_BF, HYBRID_BATCHES):
            got = hybrid(g, qd, rd, 4096, fl, order=order, policy=policy)
            assert check_rows(got, exp, 4096) == nq
            modes, flags = got[3], got[4]
            if policy == HYBRID_BATCHES and dense:
                assert (modes == HYBRID_BATCHES).all() and _path(g) == dense
                assert (flags == 1).sum() >= nq // 2, flags  # broad or narrow, the filtered pass proves most queries
            elif policy == HYBRID_ADHOC_BF or not dense:
                assert (modes == HYBRID_ADHOC_BF).all() and _path(g) == 0 and (flags == 0).all()
            else:  # automatic: 70K rows, 32 queries, filters up to 100 %: the gathers would read more than the pass
                assert (modes == HYBRID_BATCHES).all() and _path(g) == dense
    assert g.debug_info()["LAST_SEARCH_MODE"] == "RANGE_QUERY"


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(ol.F32, ol.IP), (ol.I8, ol.IP), (ol.F32, ol.L2), (ol.U8, ol.L2)])
def test_edge_radii(mode1, vtype, metric):
    """-0, +0, NaN and +inf radii next to radii at filtered neighbours (negative ones on inner product), with caps above the
    counts and with no count pointers.  Filters of at most ~700 docIds: each answer is also the row of TopKFilteredBatchDevice at
    k = 1024 cut at the radius, which holds where the whole corpus's answer is too long to restrict."""
    import torch

    rng = np.random.default_rng(5)
    n, dim, nq = 70_000, 64, 24
    g, deleted = _index(vtype, metric, n, dim)
    qs = ol.synth_rows(vtype, 9, 0, nq, dim)
    filters = _filters(rng, n, nq, deleted, ["lt10", 0.001, 0.01])
    caps = [len(f) + 50 * (i % 3) for i, f in enumerate(filters)]
    base = _radii(g, qs, Filters(filters))
    edge = [-0.0, 0.0, np.nan, np.inf]
    radii = np.array([edge[(i // 2) % len(edge)] if i % 2 else base[i] for i in range(nq)], dtype=np.float32)
    if metric == ol.IP:
        assert (radii[::2] < 0).any()  # inner-product distances below zero are answered as given
    qd, rd = _stage(g, qs), _dev(radii)
    fx = Filters(filters)
    tl, ts, tc, rc = g.topk_filtered_batch_device(qd, 1024, fx.ptrs, fx.caps, counts=fx.cptrs)
    assert rc == 0
    torch.cuda.synchronize()
    tl, ts, tc = tl.cpu().numpy(), ts.cpu().numpy(), tc.cpu().numpy()
    for exact_caps in (False, True):
        fl = Filters(filters, caps=None if exact_caps else caps, exact_caps=exact_caps)
        for order in (BY_SCORE, BY_ID):
            exp = []
            for i in range(nq):
                L, S = tl[i, : tc[i]], ts[i, : tc[i]]
                m = S <= radii[i]
                L, S = L[m], S[m]
                o = np.argsort(L, kind="stable") if order == BY_ID else np.arange(len(L))
                exp.append((L[o], S[o]))
            label_rows = want(g, qd, rd, filters, order)
            for i, e in enumerate(label_rows):
                if e is not None:
                    assert e[0].tolist() == exp[i][0].tolist() and e[1].tobytes() == exp[i][1].tobytes(), i
            for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
                got = hybrid(g, qd, rd, 4096, fl, order=order, policy=policy)
                assert check_rows(got, exp, 4096) == nq
                if policy == HYBRID_BATCHES:
                    assert _path(g) == (1 if vtype == ol.F32 else 2)
                    if vtype == ol.F32:  # a bound that is not finite is never proven: the gather answers
                        assert all(got[4][i] == 0 for i in range(nq) if not np.isfinite(radii[i])), got[4]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(ol.F32, ol.COS), (ol.I8, ol.L2)])
@pytest.mark.parametrize("cap", [1, 16, 4096])
def test_counts_past_cap(mode1, vtype, metric, cap):
    rng = np.random.default_rng(cap)
    n, dim, nq = 70_000, 128, 20
    g, deleted = _index(vtype, metric, n, dim)
    qs = ol.synth_rows(vtype, 11, 0, nq, dim)
    filters = _filters(rng, n, nq, deleted, [0.01, 0.1, 0.5, 1.0])
    fl = Filters(filters)
    radii = _radii(g, qs, fl, ranks=(10, 100, 1000))
    qd, rd = _stage(g, qs), _dev(radii)
    for order in (BY_SCORE, BY_ID):
        exp = want(g, qd, rd, filters, order)
        for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
            got = hybrid(g, qd, rd, cap, fl, order=order, policy=policy)
            assert check_rows(got, exp, cap) == nq
            if cap < 4096:
                assert (got[2] > cap).any()


@pytest.mark.gpu
def test_overflowed_dense_query_is_answered_by_the_gather(mode1):
    """clustered_corpus block A: 40,000 copies at one distance from qa.  3,500 of them in qa's filter at a radius above that
    distance overflow the filtered main pass's lists (256 queries: about 33 row ranges of 96 entries); the gather answers it
    with flag 0, every copy at the same score bits, the other queries stay on the dense route."""
    from test_vecsim_large_k_batch import clustered_corpus

    vs = mode1
    rng = np.random.default_rng(31)
    n, dim, nq = 70_000, 128, 256
    rows, qa, qb = clustered_corpus(n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == len(rows)
    qs = ol.synth_rows(ol.F32, 12, 0, nq, dim)
    qs[0] = qa
    filters = _filters(rng, n, nq, [], [0.01, 0.1])
    filters[0] = np.sort(rng.choice(np.arange(n + 1, n + 40_001), 3500, replace=False)).astype(np.uint32)
    fl = Filters(filters)
    radii = _radii(g, qs, fl, ranks=(10, 100))
    radii[0] = np.float32(0.31)
    qd, rd = _stage(g, qs), _dev(radii)
    got = hybrid(g, qd, rd, 4096, fl, order=BY_ID, policy=HYBRID_BATCHES)
    assert _path(g) == 1 and got[4][0] == 0 and (got[4][1:] == 1).sum() >= nq - 5, got[4][:8]
    assert got[2][0] == 3500 and got[0][0, :3500].tolist() == filters[0].astype(np.int64).tolist()
    one = hybrid(g, qd[:1], rd[:1], 4096, Filters([filters[0][:1]]), policy=HYBRID_ADHOC_BF)
    assert len(set(got[1][0, :3500].view(np.uint32).tolist())) == 1 and got[1][0, 0].tobytes() == one[1][0, 0].tobytes()
    exp = want(g, qd, rd, filters, BY_ID)
    assert check_rows(got, exp, 4096, skip_unknown=True) >= nq - 5


@pytest.mark.gpu
def test_nan_rows_of_multi_value_labels(mode1):
    """L2, three rows per docId, one row with a NaN component in each position: the answer keeps the smallest passing row"""
    vs = mode1
    dim = 16
    rng = np.random.default_rng(8)
    q = rng.standard_normal(dim).astype(np.float32)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2, multi=True)
    for lab in range(1, 301):
        near = q + 0.05 * rng.standard_normal(dim).astype(np.float32)
        far = q + 0.5 * rng.standard_normal(dim).astype(np.float32)
        bad = rng.standard_normal(dim).astype(np.float32)
        bad[lab % dim] = np.nan
        rows = [[bad, near, far], [near, bad, far], [near, far, bad], [far, near, far]][lab % 4]
        for r in rows:
            g.add(r, lab)
    qs = np.repeat(q[None, :], 4, axis=0)
    radii = np.array([0.1, 1.0, 10.0, 1e9], dtype=np.float32)
    filters = [np.arange(1, 301, dtype=np.uint32), np.arange(1, 301, 2, dtype=np.uint32), np.arange(5, 400, dtype=np.uint32),
               np.array([4, 8, 9, 10], dtype=np.uint32)]
    fl = Filters(filters)
    qd, rd = _stage(g, qs), _dev(radii)
    for order in (BY_SCORE, BY_ID):
        exp = want(g, qd, rd, filters, order)
        got = hybrid(g, qd, rd, 4096, fl, order=order, policy=HYBRID_BATCHES)
        assert check_rows(got, exp, 4096) == 4 and _path(g) == 0
        # at the widest radius every label has a passing row, whichever of its rows is NaN
        assert got[2][3] == 4 and got[2][2] == 296
        # the smallest passing row: near rows everywhere but in the last pattern, whose near row sits between two far ones
        assert (got[1][1, : got[2][1]] < 1.0).all()


@pytest.mark.gpu
def test_pending_filters_no_host_wait_and_launch_counts(mode1):
    """AND / OR results of the device posting-list batches feed the call while pending; the call returns while the caller's
    stream is still spinning; the launch count is the same at 16 and 256 queries"""
    import torch
    from redisearch_b200 import postings as ps

    vs = mode1
    rng = np.random.default_rng(24)
    n, dim = 70_000, 64
    g, _ = _index(ol.F32, ol.COS, n, dim, deletes=False)
    pool = [np.sort(rng.choice(np.arange(1, n + 1), s, replace=False)).astype(np.uint64) for s in (30_000, 20_000, 10_000)]
    pls = [ps.PostingList.from_arrays(p) for p in pool]
    nq = 16
    batch = [[pls[i % 3], pls[(i + 1) % 3]] for i in range(nq)]
    qs = ol.synth_rows(ol.F32, 16, 0, nq, dim)
    qd = _stage(g, qs)
    rd = _dev(_radii(g, qs, Filters([np.arange(1, n + 1, dtype=np.uint32)] * nq), ranks=(100, 1000)))
    for kind in ("and", "or"):
        res = ps.intersect_batch_device(batch) if kind == "and" else ps.union_batch_device(batch)
        for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
            lab, sc, cnt, md, rc = g.hybrid_range_batch_device(qd, rd, 4096, [r[1] for r in res], [r[3] for r in res],
                                                               counts=[r[2] for r in res], params=_params(policy))
            assert rc == 0
            torch.cuda.synchronize()
            fn = np.intersect1d if kind == "and" else np.union1d
            filters = [fn(pool[i % 3], pool[(i + 1) % 3]).astype(np.uint32) for i in range(nq)]
            exp = want(g, qd, rd, filters, BY_SCORE)
            assert check_rows((lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().astype(np.int64)), exp, 4096) == nq
        for r in res:
            r[0].free_after(None)
    # launches: 2 on the gather, 8 on the fp32 route over unit rows, whatever nq
    for policy, expect in ((HYBRID_ADHOC_BF, 2), (HYBRID_BATCHES, 8)):
        launches = []
        for m in (16, 256):
            qs2 = ol.synth_rows(ol.F32, 17, 0, m, dim)
            filters = _filters(rng, n, m, [], [0.01, 0.5])
            fl = Filters(filters)
            qd2, rd2 = _stage(g, qs2), _dev(np.full(m, 0.7, dtype=np.float32))
            hybrid(g, qd2, rd2, 256, fl, policy=policy)  # warm-up
            g.stats(reset=True)
            hybrid(g, qd2, rd2, 256, fl, policy=policy)
            launches.append(g.stats(reset=True).kernel_launches)
        assert launches[0] == launches[1] == expect, (policy, launches)
    # no host wait
    fl = Filters(_filters(rng, n, nq, [], [0.01, 0.5]))
    out_l = torch.empty((nq, 256), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, 256), dtype=torch.float32, device="cuda")
    out_c = torch.empty(nq, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
        def run():
            return g.hybrid_range_batch_device(qd, rd, 256, fl.ptrs, fl.caps, counts=fl.cptrs, params=_params(policy), out_labels=out_l,
                                               out_scores=out_s, out_counts=out_c, stream=s)[4]

        assert run() == 0
        s.synchronize()
        ref = (out_l.cpu().numpy().copy(), out_s.cpu().numpy().copy())
        out_l.fill_(7)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(200_000_000)
        assert run() == 0
        busy = not s.query()
        s.synchronize()
        assert busy, "the call waited for the caller's stream"
        assert out_l.cpu().numpy().tolist() == ref[0].tolist() and out_s.cpu().numpy().tobytes() == ref[1].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(ol.F32, ol.L2), (ol.I8, ol.COS)])
def test_mutations_and_interleaving_on_one_stream(mode1, vtype, metric):
    """deletes, re-adds and new rows between calls show up in the next call; other device batches enqueued on the same stream
    between two calls leave both answers intact"""
    import torch

    rng = np.random.default_rng(41)
    n, dim, nq = 70_000, 64, 16
    g, deleted = _index(vtype, metric, n, dim)
    qs = ol.synth_rows(vtype, 13, 0, nq, dim)
    filters = _filters(rng, n, nq, deleted, [0.05, 0.5])
    fl = Filters(filters)
    qd = _stage(g, qs)
    rd = _dev(_radii(g, qs, fl, ranks=(100, 1000)))
    s = torch.cuda.Stream()
    for stage in range(3):
        if stage == 1:
            for d in filters[0][:50].tolist():
                g.delete(int(d))
        if stage == 2:
            extra = ol.synth_rows(vtype, 14, 0, 300, dim)
            for j, r in enumerate(extra):
                assert g.add(r, int(filters[j % nq][-1]) if j % 2 else n + 1 + j) >= 0
            g.add(qs[0], int(filters[0][0]))
        for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
            lab, sc, cnt, md, rc = g.hybrid_range_batch_device(qd, rd, 4096, fl.ptrs, fl.caps, counts=fl.cptrs, params=_params(policy),
                                                               stream=s)
            assert rc == 0
            # another device batch on the same stream before the answer is read
            ol_, os_, oc_, rc3 = g.label_range_batch_device(qd, rd, 64, BY_ID, stream=s)
            lab3, sc3, cnt3, md3, rc4 = g.hybrid_range_batch_device(qd, rd, 4096, fl.ptrs, fl.caps, counts=fl.cptrs, order=BY_ID,
                                                                    params=_params(policy), stream=s)
            assert rc3 == 0 and rc4 == 0
            s.synchronize()
            check_rows((lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().astype(np.int64)), want(g, qd, rd, filters, BY_SCORE), 4096)
            check_rows((lab3.cpu().numpy(), sc3.cpu().numpy(), cnt3.cpu().numpy().astype(np.int64)), want(g, qd, rd, filters, BY_ID), 4096)


@pytest.mark.gpu
def test_limits(mode1):
    import torch

    vs = mode1
    g, _ = _index(ol.F32, ol.COS, 2000, 32, deletes=False)
    qs = ol.synth_rows(ol.F32, 3, 0, 2, 32)
    qd, rd = _stage(g, qs), _dev(np.array([0.5, 0.5], dtype=np.float32))
    fl = Filters([np.arange(1, 100, dtype=np.uint32)] * 2)

    def call(cap=16, order=BY_SCORE, policy=None, caps=None, nq=2, idx=g):
        lab = torch.empty((max(nq, 1), max(cap, 1)), dtype=torch.int64, device="cuda")
        sc = torch.empty((max(nq, 1), max(cap, 1)), dtype=torch.float32, device="cuda")
        cn = torch.empty(max(nq, 1), dtype=torch.int32, device="cuda")
        return idx.hybrid_range_batch_device(qd[:nq], rd, cap, fl.ptrs[:nq], caps if caps is not None else fl.caps[:nq],
                                             counts=fl.cptrs[:nq], order=order, params=_params(policy), out_labels=lab, out_scores=sc,
                                             out_counts=cn)[4]

    assert call(cap=0) == -1 and call(cap=4097) == -1 and call(order=2) == -1 and call(policy=5) == -1
    assert call(policy=1) == -1  # STANDARD_KNN is no hybrid policy
    assert call(nq=0) == 0 and call(cap=4096) == 0
    assert call(caps=[99, 0x1_0000_0000]) == -2
    torch.cuda.synchronize()
    assert g.debug_info()["LAST_SEARCH_MODE"] == "RANGE_QUERY"
    sparse = vs.VecSimIndex(vs.VecSimType_FLOAT32, 32, vs.VecSimMetric_Cosine, multi=True)
    rows = ol.synth_rows(ol.F32, 4, 0, 4, 32)
    for j, r in enumerate(rows):
        assert sparse.add(r, (1 << 40) + j) == 1
    assert call(idx=sparse) == -2


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(ol.F32, ol.L2), (ol.I8, ol.L2), (ol.U8, ol.L2)])
def test_eight_queries_against_the_reference(mode1, vtype, metric):
    """rows read back from HBM into the reference (or its C restatement): its range answer intersected with the filter"""
    vs = mode1
    rng = np.random.default_rng(61)
    n, dim, nq = 70_000, 64, 16
    g, _ = _index(vtype, metric, n, dim, deletes=False)
    stored = np.zeros(n * g.L.VecSimParams_GetQueryBlobSize(g.vtype, dim, g.metric), dtype=np.uint8)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, stored.ctypes.data_as(C.c_void_p)) == 0
    rows = stored.view(ol.synth_rows(vtype, 1, 0, 1, dim).dtype).reshape(n, dim)
    o = ol.RefIndex(vtype, dim, metric) if ol.ref_vecsim() is not None else ol.PortIndex(vtype, dim, metric, tier=ol.TIER_AVX512)
    o.add_many(rows, 1)
    qs = ol.synth_rows(vtype, 62, 0, nq, dim)
    filters = _filters(rng, n, nq, [], [0.01, 0.1, 0.5])
    fl = Filters(filters)
    radii = _radii(g, qs, fl, ranks=(10, 100, 1000))
    qd, rd = _stage(g, qs), _dev(radii)
    for policy in (HYBRID_ADHOC_BF, HYBRID_BATCHES):
        lab, sc, cnt, modes, flags = hybrid(g, qd, rd, 4096, fl, order=BY_ID, policy=policy)
        for i in range(0, nq, 2):
            ei, es = o.range(qs[i], float(radii[i]), BY_ID)
            m = np.isin(ei, filters[i].astype(np.int64))
            ei, es = ei[m], es[m].astype(np.float32)
            assert cnt[i] == len(ei), (i, cnt[i], len(ei))
            assert lab[i, : len(ei)].tolist() == ei.tolist() and sc[i, : len(ei)].tobytes() == es.tobytes(), i
