"""VecSimB200_RangeQueryBatchDevice: range batches with device pointers end to end (DESIGN.md §4.11).

Routes: the fp32 route of VecSimB200_RangeQueryBatch with the hits written into each query's `cap` slots; a fixed-radius pass on
the s8 / u8 tensor cores for int8 / uint8 batches (coarse_wgmma_kernel<true, 8, kOp, 1, V>, kOp 1 / 2 / 4), whose distances are
the reference's floats; the exact scan on the device for everything else and for every query a route could not complete.  One
CTA per query then orders the hits as finish_reply does and maps rows to labels.

CPU: the 8-bit admission rule and its integer pre-test (range_int_bound in coarse_tc.cu), restated from the kernel's constants,
keep exactly the rows whose float distance is <= the radius; the restated sort order is finish_reply's.
GPU: every answer equals VecSimIndex_RangeQuery per query (labels, float32 score bits and order, both orders); radii the host
API refuses (negative inner-product radii) are checked against the C restatement of the reference.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol

_VT = {ol.F32: 0, ol.F16: 3, ol.BF16: 2, ol.I8: 4, ol.U8: 5}  # VecSimType
_MT = {ol.L2: 0, ol.IP: 1, ol.COS: 2}                          # VecSimMetric
BY_ID, BY_SCORE = 0, 1
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
# restated from coarse_tc.cu: range_int_bound clamps at +-2^30; the cosine pre-test's margin (fthr_dot)
BOUND_CLAMP = 1073741824.0
COS_MARGIN = 1e-6


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


# ------------------------------------------------------------------------------------------------------------------
# CPU: the admission rule and the pre-tests, restated
# ------------------------------------------------------------------------------------------------------------------
def f32(x):
    return np.float32(x)


def int_bound(r):
    """range_int_bound: the largest integer x with float(x) <= r (clamped)."""
    r = f32(r)
    if np.isnan(r) or r < f32(-BOUND_CLAMP):
        return INT_MIN
    if r >= f32(BOUND_CLAMP):
        return INT_MAX
    x = int(np.floor(r))
    while f32(x + 1) <= r:
        x += 1
    return x


def _radii():
    out = [0.0, -0.0, np.nextafter(f32(0), f32(1)), -np.nextafter(f32(0), f32(1)), np.float32(1.17549435e-38) / 4]
    for v in (1, 2, 7, 100, 4095, 65025, 2 ** 23 + 1, 123456789, 2 ** 28 + 3, 5 * 2 ** 26):
        for s in (1, -1):
            x = f32(s * v)
            out += [x, np.nextafter(x, f32(np.inf)), np.nextafter(x, f32(-np.inf))]
    out += [f32(2 ** 24 + 1), f32(2 ** 24 - 1), f32(2 ** 24), f32(-(2 ** 24 + 1))]
    out += [np.finfo(np.float32).max, -np.finfo(np.float32).max, np.inf, -np.inf, np.nan]
    return [f32(r) for r in out]


def _window(r):
    c = 0 if not np.isfinite(r) else int(np.clip(np.floor(r), -2 ** 29, 2 ** 29))
    return range(c - 80, c + 81)


@pytest.mark.parametrize("op", ["ip", "l2"])
def test_integer_pretest_is_the_float_test(op):
    """Inner product (x = 1 - dot) and L2 (x = e, the int32 distance): x <= range_int_bound(r) iff float(x) <= r, over every
    integer in a window around each radius (a NaN radius keeps nothing, +inf everything)."""
    for r in _radii():
        X = int_bound(r)
        for x in _window(r):
            if op == "l2" and x < 0:
                continue
            want = bool(f32(x) <= r)  # the kernel's exact test on the float distance
            assert (x <= X) == want, (float(r), x, X)
        if np.isnan(r):
            assert X == INT_MIN
    # integers that round to the same float as the radius are all kept
    r = f32(2 ** 24 + 4)
    assert int_bound(r) == 2 ** 24 + 5 and f32(2 ** 24 + 5) == r


def _cos_d(dot, nr, nq):
    """the kernel's cosine distance: 1 - fl(fl(dot) / fl(nr nq))"""
    return f32(f32(1) - f32(f32(dot) / f32(f32(nr) * f32(nq))))


def _cos_pre(dot, nr, nq, r):
    t = f32(f32(nq) * f32(f32(f32(1) - r) - f32(f32(COS_MARGIN) * f32(f32(1) + abs(r)))))
    return bool(f32(dot) >= f32(f32(nr) * t))


def test_cosine_pretest_is_conservative():
    """int8 / uint8 cosine: the float pre-test never drops a row the exact test d <= r keeps, over rows of real norms (the dot
    product bounded by Cauchy-Schwarz) and radii around the distances they produce."""
    rng = np.random.default_rng(3)
    with np.errstate(all="ignore"):
        for dim in (32, 768, 2048):
            for _ in range(200):
                lo, hi = (-128, 127) if rng.integers(2) else (0, 255)
                q = rng.integers(lo, hi + 1, dim).astype(np.int64)
                rows = rng.integers(lo, hi + 1, (8, dim)).astype(np.int64)
                rows[0] = q  # distance ~0
                rows[1] = -q if lo < 0 else q // 2
                nq = f32(np.sqrt(f32((q * q).sum())))
                for a in rows:
                    dot = int(a @ q)
                    nr = f32(np.sqrt(f32((a * a).sum())))
                    d = _cos_d(dot, nr, nq)
                    for r in (d, np.nextafter(d, f32(np.inf)), np.nextafter(d, f32(-np.inf)), f32(0), f32(-0.0), f32(1), f32(2)):
                        if d <= r:
                            assert _cos_pre(dot, nr, nq, r), (dim, dot, float(nr), float(nq), float(r))
        # a zero row: NaN distance, never kept (the pre-test may pass it: the exact test decides)
        assert not (_cos_d(0, 0.0, 5.0) <= f32(np.inf))


def _finish_order(keys, labels, by_id):
    """range_finish_kernel's comparison, restated"""
    idx = list(range(len(keys)))
    if by_id:
        return sorted(idx, key=lambda i: (labels[i], keys[i]))
    return sorted(idx, key=lambda i: (keys[i], labels[i]))


def _orderable_key(x):
    x = f32(x) + f32(0.0)
    u = int(np.array([x], dtype=np.float32).view(np.uint32)[0])
    return (~u) & 0xFFFFFFFF if u & 0x80000000 else u | 0x80000000


def test_sort_order_is_finish_replys_on_ties():
    """BY_SCORE: (score, label), with -0 and +0 equal; BY_ID: label — the order finish_reply gives."""
    rng = np.random.default_rng(1)
    scores = f32(rng.integers(-3, 4, 300)) * f32(0.5)
    scores[::7] = f32(-0.0)
    labels = rng.permutation(10_000)[:300]
    keys = [_orderable_key(s) for s in scores]
    want_score = sorted(range(300), key=lambda i: (float(scores[i]), labels[i]))
    assert _finish_order(keys, labels, False) == want_score
    assert _finish_order(keys, labels, True) == sorted(range(300), key=lambda i: labels[i])


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def mode1():
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    yield vs
    vs.lib().VecSimB200_SetCoarseMode(-1)


def _index(vtype, metric, dim, rows, port=False):
    vs = _vs()
    g = vs.VecSimIndex(_VT[vtype], dim, _MT[metric])
    assert g.add_many(rows, label0=1) == len(rows)
    p = None
    if port:
        p = ol.PortIndex(vtype, dim, metric, tier=ol.TIER_AVX512)
        p.add_many(rows, 1)
    return g, p


def _stage(g, qs):
    """stored-form queries, query_pitch() apart, as a CUDA tensor"""
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


def _run(g, qs, radii, cap, order, stream=None):
    import torch

    d_q = _stage(g, qs)
    d_r = torch.from_numpy(np.ascontiguousarray(radii, dtype=np.float32)).cuda()
    lab, sc, cnt, rc = g.range_batch_device(d_q, d_r, cap, order, stream=stream)
    torch.cuda.synchronize()
    assert rc == 0
    return lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def _flags(g, nq):
    f = np.zeros(nq, dtype=np.uint32)
    assert _vs().lib().VecSimB200_LastCoarseFlags(g.h, f.ctypes.data_as(C.c_void_p), nq) == 0
    return f


def _path(g):
    return _vs().lib().VecSimB200_LastBatchPath(g.h)


def _check(g, p, qs, radii, cap, order, lab, sc, cnt, expect_full=True):
    for i in range(qs.shape[0]):
        r = float(radii[i])
        if r >= 0 or np.isnan(r):
            if np.isnan(r):
                ei, es = np.zeros(0, np.int64), np.zeros(0)
            else:
                ei, es, code = g.range(qs[i], r, order)
                assert code == 0
            ties = False
        else:  # the host API refuses a negative radius: the C restatement of the reference
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
    rows = ol.synth_rows(ol.F32, 7, 0, n, dim)
    g, _ = _index(ol.F32, metric, dim, rows)
    qs = ol.synth_rows(ol.F32, 8, 0, nq, dim)
    if metric == ol.IP:
        qs = (qs.astype(np.float64) / dim).astype(np.float32)  # distances 1 - dot stay positive
    radii = _radii_at(g, qs, [1, 10, 100, 37])
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 128, order)
        assert _path(g) == 1 and _flags(g, nq).tolist() == [1] * nq
        _check(g, None, qs, radii, 128, order, lab, sc, cnt)


_EIGHT = [(d, nq) for d, nq in ((32, 16), (128, 64), (768, 300), (2048, 16))]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("metric", [ol.IP, ol.COS, ol.L2])
@pytest.mark.parametrize("dim,nq", _EIGHT)
def test_8bit_route(mode1, vtype, metric, dim, nq):
    n = 70_000
    rows = ol.synth_rows(vtype, 11, 0, n, dim)
    rows[3000:3010] = rows[100]  # ties: ten copies of one row
    g, p = _index(vtype, metric, dim, rows, port=True)
    qs = ol.synth_rows(vtype, 12, 0, nq, dim)
    qs[0] = rows[100]  # a query equal to the copies
    radii = _radii_at(g, qs, [10, 100])
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 256, order)
        assert _path(g) == 2 and _flags(g, nq).tolist() == [1] * nq, (_path(g), _flags(g, nq)[:8])
        _check(g, p, qs, radii, 256, order, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("metric", [ol.COS, ol.L2])
def test_8bit_reference_scan(mode1, vtype, metric):
    """a few queries against the reference's own compiled range scan"""
    if ol.ref_vecsim() is None:
        pytest.skip("oracle/_ref is not built")
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(vtype, 21, 0, n, dim)
    g, _ = _index(vtype, metric, dim, rows)
    ref = ol.RefIndex(vtype, dim, metric)
    ref.add_many(rows, 1)
    qs = ol.synth_rows(vtype, 22, 0, nq, dim)
    radii = _radii_at(g, qs, [10, 50])
    lab, sc, cnt = _run(g, qs, radii, 256, BY_ID)
    assert _path(g) == 2
    for i in range(4):
        ri, rs = ref.range(qs[i], float(radii[i]), BY_ID)
        assert int(cnt[i]) == len(ri)
        assert lab[i, :len(ri)].tolist() == ri.tolist()
        assert sc[i, :len(ri)].astype(np.float32).tobytes() == rs.astype(np.float32).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_edge_radii(mode1, vtype):
    """L2, many rows at one distance: a radius there returns all of them, one float below none; 0.0 and -0.0 with copies of the
    query; a NaN radius keeps nothing; +inf with a small cap gives the true count and a padded row; count == cap is written
    whole and cap + 1 pads."""
    dim, n = 64, 70_000
    rows = ol.synth_rows(vtype, 31, 0, n, dim)
    q = rows[500].copy()
    far = q.copy()
    far[:3] = np.where(q[:3].astype(np.int64) < 100, q[:3].astype(np.int64) + 1, q[:3].astype(np.int64) - 1).astype(q.dtype)
    rows[20_000:20_040] = q  # 40 copies of the query (distance 0)
    rows[40_000:40_101] = far  # 101 rows at one shared distance (3)
    g, p = _index(vtype, ol.L2, dim, rows, port=True)
    d_far = f32(float(((q.astype(np.int64) - far.astype(np.int64)) ** 2).sum()))
    nq = 16
    qs = np.repeat(q[None], nq, axis=0)
    radii = np.array([d_far, np.nextafter(d_far, f32(-np.inf)), 0.0, -0.0, np.nan, np.inf] + [d_far] * 10, dtype=np.float32)
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 256, order)
        _check(g, p, qs[:4], radii[:4], 256, order, lab, sc, cnt)
        assert cnt[4] == 0 and (lab[4] == -1).all()
        assert cnt[5] == n and (lab[5] == -1).all() and np.isnan(sc[5]).all()
        assert int(cnt[0]) == 142 and int(cnt[1]) == 41 and int(cnt[2]) == int(cnt[3]) == 41
    n0 = int(cnt[2])  # hits at radius 0: the copies of the query
    for cap, full in ((n0, True), (n0 - 1, False)):
        lab, sc, cnt = _run(g, qs[2:3], radii[2:3], cap, BY_SCORE)
        assert int(cnt[0]) == n0
        if full:
            assert (lab[0] != -1).all() and (sc[0] == 0).all()
        else:
            assert (lab[0] == -1).all() and np.isnan(sc[0]).all()


@pytest.mark.gpu
def test_cosine_zero_row_never_returned(mode1):
    dim, n = 128, 70_000
    rows = ol.synth_rows(ol.I8, 41, 0, n, dim)
    rows[777] = 0
    g, p = _index(ol.I8, ol.COS, dim, rows)
    qs = ol.synth_rows(ol.I8, 42, 0, 16, dim)
    radii = _radii_at(g, qs, [50])
    radii[:4] = np.inf  # every row but the zero row (its NaN distance never passes)
    lab, sc, cnt = _run(g, qs, radii, 4096, BY_ID)
    assert _path(g) == 2
    assert cnt[:4].tolist() == [n - 1] * 4
    for i in range(4, 16):
        assert 778 not in lab[i, :int(cnt[i])].tolist()
    _check(g, p, qs, radii, 4096, BY_ID, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_list_overflow_takes_the_exact_scan(mode1, vtype):
    """more than 256 hits in one row range (near-duplicates stored together): those queries report flag 0 and still give the
    same answer; the rest keep flag 1"""
    dim, n = 128, 70_000
    rows = ol.synth_rows(vtype, 51, 0, n, dim)
    base = rows[10].copy()
    base[0] = 50
    # 40,000 near-duplicates in a row: every row range holds more than 256 of them
    rows[20_000:60_000] = base
    rows[20_000:60_000, 0] = 50 + np.arange(40_000) % 3
    g, _ = _index(vtype, ol.L2, dim, rows)
    qs = ol.synth_rows(vtype, 52, 0, 16, dim)
    qs[3] = base
    radii = _radii_at(g, qs, [10])
    radii[3] = 400.0
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 1024, order)
        f = _flags(g, 16)
        assert f[3] == 0 and f.sum() == 15 and _path(g) == 2
        assert cnt[3] >= 40_000 and (lab[3] == -1).all()
        _check(g, None, qs, radii, 1024, order, lab, sc, cnt)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["f16", "bf16", "mode0", "mode2_f32", "small", "nq15"])
def test_batches_off_the_routes(case):
    vs = _vs()
    vtype, metric, dim, n, nq = ol.I8, ol.L2, 64, 70_000, 16
    mode = 1
    if case in ("f16", "bf16"):  # L2: radii >= 0, so VecSimIndex_RangeQuery on the same index is the yardstick
        vtype = ol.F16 if case == "f16" else ol.BF16
    elif case == "mode0":
        mode = 0
    elif case == "mode2_f32":
        vtype, metric, mode = ol.F32, ol.L2, 2
    elif case == "small":
        n = 20_000
    else:
        nq = 15
    vs.lib().VecSimB200_SetCoarseMode(mode)
    try:
        rows = ol.synth_rows(vtype, 61, 0, n, dim)
        g, p = _index(vtype, metric, dim, rows, port=True)
        qs = ol.synth_rows(vtype, 62, 0, nq, dim)
        radii = _radii_at(g, qs, [20])
        for order in (BY_SCORE, BY_ID):
            lab, sc, cnt = _run(g, qs, radii, 512, order)
            assert _path(g) == 0 and _flags(g, nq).tolist() == [0] * nq
            _check(g, p, qs, radii, 512, order, lab, sc, cnt)
    finally:
        vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.F32])
def test_mutations_between_batches(mode1, vtype):
    """appends, raw in-place overwrites and swap-deletes between two batches (the int32 |row|^2 table of 8-bit L2 indexes, the
    fp16 shadow of fp32 ones)"""
    dim, n, nq = 128, 70_000, 16
    rows = ol.synth_rows(vtype, 71, 0, n, dim)
    g, _ = _index(vtype, ol.L2, dim, rows)
    qs = ol.synth_rows(vtype, 72, 0, nq, dim)
    radii = _radii_at(g, qs, [10])
    _run(g, qs, radii, 256, BY_SCORE)
    extra = ol.synth_rows(vtype, 73, 0, 300, dim)
    g.add_many(extra, label0=n + 1)
    for i in range(0, nq, 2):
        g.add(qs[i], 5 + i)  # overwrite label 5 + i in place with the query itself (distance 0)
    for lab_ in (8, 9_000, 40_001):
        g.delete(lab_)
    for order in (BY_SCORE, BY_ID):
        lab, sc, cnt = _run(g, qs, radii, 256, order)
        assert _path(g) == (2 if vtype == ol.I8 else 1)
        _check(g, None, qs, radii, 256, order, lab, sc, cnt)
        assert all(5 + i in lab[i, :int(cnt[i])].tolist() for i in range(0, nq, 2) if int(cnt[i]) <= 256)


@pytest.mark.gpu
def test_outputs_feed_torch_on_the_callers_stream(mode1):
    import torch

    dim, n, nq = 128, 70_000, 64
    rows = ol.synth_rows(ol.I8, 81, 0, n, dim)
    g, _ = _index(ol.I8, ol.IP, dim, rows)
    qs = ol.synth_rows(ol.I8, 82, 0, nq, dim)
    labels, scores, rc = g.topk_batch(qs, 10)
    radii = scores[:, 9].astype(np.float32)
    s = torch.cuda.Stream()
    d_q = _stage(g, qs)
    d_r = torch.from_numpy(radii).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        lab, sc, cnt, rc = g.range_batch_device(d_q, d_r, 64, BY_SCORE, stream=s)
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
    rows = ol.synth_rows(ol.F32, 91, 0, 1000, dim)
    g, _ = _index(ol.F32, ol.L2, dim, rows)
    qs = ol.synth_rows(ol.F32, 92, 0, 4, dim)
    d_q, d_r = _stage(g, qs), torch.ones(4, device="cuda")
    for cap, order in ((0, BY_SCORE), (4097, BY_SCORE), (16, 7)):
        out = torch.empty((4, max(cap, 1)), dtype=torch.int64, device="cuda")
        outs = torch.empty((4, max(cap, 1)), dtype=torch.float32, device="cuda")
        assert g.range_batch_device(d_q, d_r, cap, order, out_labels=out, out_scores=outs)[3] == -1
    assert g.range_batch_device(d_q[:0], d_r[:0], 16)[3] == 0
    m = vs.VecSimIndex(0, dim, 0, multi=True)
    m.add_many(rows, label0=1)
    assert m.range_batch_device(d_q, d_r, 16)[3] == -1
    torch.cuda.synchronize()
