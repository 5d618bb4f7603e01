"""fp16 / bf16 range batches on the tensor cores (DESIGN.md §4.11): VecSimB200_RangeQueryBatchDevice and
VecSimB200_LabelRangeQueryBatchDevice on inner-product / cosine indexes of 16-bit rows.

The route runs the direct 16-bit fixed-bound pass with T_q = radius_q + eps16_q, rescores every kept row with DistTile16 (the
CUDA-core arithmetic of the exact scan) and keeps it iff d <= radius_q.  eps16_q bounds |tc - cc| between the wgmma distance and
the CUDA-core one, so a row the pass drops is outside the radius and a query whose lists did not overflow gets the exact scan's
answer bit for bit.

CPU: eps16_q restated in float64 from the constants in coarse_tc.cu, held to at least twice B_tc + B_cc (the bounds of
test_half_precision_bounds.py) at the worst-case magnitude X |q|, and never finite where X or |q| is not.
GPU: every batch equals the same batch under SetCoarseMode(0) and VecSimIndex_RangeQuery per query (labels, score bits, counts,
order, cap rule), with LastBatchPath 2 and the per-query flags of the route.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import oracle_lib as ol
from test_half_precision_bounds import bound_cuda_core, bound_tensor_core, chain_length, decode16, to16

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "redisearch_b200", "csrc")
_VT = {ol.F16: 3, ol.BF16: 2}
_MT = {ol.IP: 1, ol.COS: 2}
BY_ID, BY_SCORE = 0, 1
WGMMA_MAX_DIM = 1024  # coarse_tc.cu wgmma_fits: the widest 16-bit dim of the direct pass
F32_MAX = float(np.finfo(np.float32).max)


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constants():
    src = _read("coarse_tc.cu")
    out = {}
    for name in ("kR16U", "kR16TcStep", "kR16Underflow", "kR16Flush", "kR16Margin", "kR16MaxMag"):
        m = re.search(r"constexpr double " + name + r"\s*=\s*([0-9a-fA-Fxp.+-]+);", src)
        assert m, name
        v = m.group(1)
        out[name] = float.fromhex(v) if "0x" in v else float(v)
    return out


K = _constants()


# ------------------------------------------------------------------------------------------------------------------
# CPU: the margin, restated
# ------------------------------------------------------------------------------------------------------------------
def up(x):
    """one step up in float64: the restatement rounds to nearest, the kernel up"""
    return np.nextafter(x, np.inf)


def x_bound(max_norm, dim):
    """X from the float sqrt of the largest fp32 |row|^2 (range_bound16_kernel)"""
    d = float(dim)
    return up(up(float(max_norm) * (1.0 + 2.0 ** -23) * up(math.sqrt(up(1.0 + d * 2.0 ** -20)))) + up(math.sqrt(d * 2.0 ** -149)))


def eps16(dim, max_norm, qn):
    """(eps16_q, M) as range_bound16_kernel computes them (float64, every step raised by one ulp)"""
    with np.errstate(all="ignore"):
        d = float(dim)
        mag = up(x_bound(max_norm, dim) * float(qn))
        chain = chain_length(dim) + 7
        gamma = up(chain * K["kR16U"] / (1.0 - chain * K["kR16U"]))
        ue = up(K["kR16U"] * up(1.0 + mag))
        b_tc = up(up(d * K["kR16TcStep"] * mag) + ue)
        b_cc = up(up(up(gamma * mag) + ue) + d * K["kR16Underflow"])
        return up(K["kR16Margin"] * up(up(b_tc + b_cc) + d * K["kR16Flush"])), mag


def thr16(dim, max_norm, qn, radius):
    """T_q as a float32, -inf where the query can never be proven"""
    e, mag = eps16(dim, max_norm, qn)
    with np.errstate(all="ignore"):
        t = up(float(np.float32(radius)) + e)  # the kernel reads the float radius
        t32 = np.float32(t)
        if np.isfinite(t32) and float(t32) < t:
            t32 = np.nextafter(t32, np.float32(np.inf))
    ok = math.isfinite(qn) and math.isfinite(x_bound(max_norm, dim)) and mag < K["kR16MaxMag"] and np.isfinite(t32)
    return t32 if ok else np.float32(-np.inf)


def test_constants_match_the_sources():
    assert K == {"kR16U": 2.0 ** -24, "kR16TcStep": 2.0 ** -22, "kR16Underflow": 2.0 ** -149, "kR16Flush": 2.0 ** -126,
                 "kR16Margin": 2.0, "kR16MaxMag": 2.0 ** 120}
    cu, host = _read("coarse_tc.cu"), _read("vecsim_index.cpp")
    # m + 7 of B_cc is test_half_precision_bounds.chain_length(dim) + 7
    assert "const double chain = 8.0 * ((dim / 8 + 31) / 32) + (double)((dim % 8 + 31) / 32) + 7.0;" in cu
    for dim in range(8, 2049, 8):
        assert 8 * ((dim // 8 + 31) // 32) + (dim % 8 + 31) // 32 == chain_length(dim)
    assert "thr[q] = ok ? t : -__int_as_float(0x7f800000);" in cu
    assert "const bool ok = isfinite(qn) && isfinite(x) && mag < kR16MaxMag && isfinite(t);" in cu
    # the route needs a finite X, and its rescoring is the 16-bit instantiation of range_refine_kernel
    assert "ensure_shadow(st) && std::isfinite(shadow_max_norm_)" in host
    assert "range_refine_kernel<DT_F16, MT_IP>" in cu and "range_refine_kernel<DT_BF16, MT_IP>" in cu


@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_margin_covers_twice_both_bounds(vtype):
    """eps16 >= 2 (B_tc + B_cc) at mag = X |q| and |e| = 1 + mag, over dims 32..1024, row and query norms from 1e-6 to the fp16
    maximum (bf16: far beyond it), and radii around zero: T_q - radius_q covers it as well."""
    norms = [1e-6, 1e-3, 0.5, 1.0, 1.0000001, 3.0, 100.0, 65504.0] + ([1e10, 1e20, 1e30] if vtype == ol.BF16 else [])
    radii = [0.0, -0.0, 1e-30, -1e-30, 1e-7, 1.0, -1.0, 2.0, -65504.0, 1e6]
    for dim in list(range(32, 257, 8)) + [512, 768, 776, 1000, WGMMA_MAX_DIM]:
        for xn in norms:
            xf = float(np.float32(xn))  # the float sqrt the kernel is given
            for qn in norms:
                e, mag = eps16(dim, xf, qn)
                if not mag < K["kR16MaxMag"]:
                    continue
                mag_true = xn * qn  # Cauchy-Schwarz: sum |x_i q_i| <= |x| |q|
                assert mag >= mag_true
                ee = 1.0 + mag_true
                need = 2.0 * (bound_tensor_core(ee, mag_true, dim) + bound_cuda_core(ee, mag_true, dim))
                assert e >= need, (dim, xn, qn, e, need)
                for r in radii:
                    t = thr16(dim, xf, qn, r)
                    if np.isfinite(t):
                        assert float(t) - float(np.float32(r)) >= need, (dim, xn, qn, r)
    # the absolute floor: tiny norms still cover the rounding of 1 - dot on both sides (2u (1 + 2u))
    e, _ = eps16(32, 1e-6, 1e-6)
    assert e >= 4 * 2.0 ** -24


def test_x_bound_covers_the_fp32_sum_of_squares():
    """max_norm is sqrtf of row_stats_kernel's fp32 sum (32 lane chains, a butterfly): x_bound lies above the exact norm"""
    rng = np.random.default_rng(5)
    for dim in (32, 128, 768, 1024):
        for scale in (1e-20, 1e-4, 1.0, 60000.0):
            for _ in range(20):
                x = (rng.uniform(-1, 1, dim) * scale).astype(np.float32)
                lanes = np.zeros(32, dtype=np.float32)
                for i in range(dim):
                    lanes[i % 32] = np.float32(np.float64(x[i]) * np.float64(x[i]) + np.float64(lanes[i % 32]))
                w = 32
                while w > 1:
                    w //= 2
                    lanes = (lanes[:w] + lanes[w:2 * w]).astype(np.float32)
                mn = np.float32(np.sqrt(lanes[0]))
                assert x_bound(mn, dim) >= math.sqrt(float(np.sum(x.astype(np.float64) ** 2))), (dim, scale)


def test_non_finite_norms_never_prove():
    for dim in (32, 768):
        for xn, qn in ((np.inf, 1.0), (np.nan, 1.0), (1.0, np.inf), (1.0, np.nan), (3e38, 3e38), (1e30, 1e20)):
            assert thr16(dim, np.float32(xn), qn, 0.5) == -np.inf, (xn, qn)
        for r in (np.inf, -np.inf, np.nan, F32_MAX):  # F32_MAX + eps rounds up to inf
            assert thr16(dim, np.float32(1.0), 1.0, r) == -np.inf, r
        assert np.isfinite(thr16(dim, np.float32(1.0), 1.0, -0.0))


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
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


_STREAM = []


def _stream():
    """one non-default stream for every call of this file"""
    import torch

    if not _STREAM:
        _STREAM.append(torch.cuda.Stream())
    return _STREAM[0]


def _index(vtype, metric, dim, rows, labels=None, multi=False):
    g = _vs().VecSimIndex(_VT[vtype], dim, _MT[metric], multi=multi)
    if labels is None:
        assert g.add_many(rows, label0=1) == len(rows)
    else:
        assert g.add_many(rows, labels=labels) == len(rows)
    return g


def _stored(g, qs):
    """stored-form blobs, query_pitch() apart (cosine: the library's own normaliser)"""
    vs = _vs()
    pitch = g.query_pitch()
    buf = np.zeros((qs.shape[0], pitch), dtype=np.uint8)
    for i in range(qs.shape[0]):
        raw = np.ascontiguousarray(qs[i]).view(np.uint8)
        buf[i, :raw.size] = raw
        if g.metric == _MT[ol.COS]:
            vs.normalize(buf[i], g.dim, g.vtype)
    return buf


def _run(g, qs, radii, cap, order, mode=1, fn="range_batch_device"):
    """one device batch on the file's stream: (labels, scores, counts, path, flags)"""
    import torch

    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(mode)
    s = _stream()
    with torch.cuda.stream(s):
        d_q = torch.from_numpy(_stored(g, qs)).cuda()
        d_r = torch.from_numpy(np.ascontiguousarray(radii, dtype=np.float32)).cuda()
        lab, sc, cnt, rc = getattr(g, fn)(d_q, d_r, cap, order, stream=s)
    s.synchronize()
    vs.lib().VecSimB200_SetCoarseMode(1)
    assert rc == 0
    nq = qs.shape[0]
    f = np.zeros(nq, dtype=np.uint32)
    assert vs.lib().VecSimB200_LastCoarseFlags(g.h, f.ctypes.data_as(C.c_void_p), nq) == 0
    return lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32), vs.lib().VecSimB200_LastBatchPath(g.h), f


def _same(a, b, what):
    assert a[0].tobytes() == b[0].tobytes(), (what, "labels")
    assert a[1].astype(np.float32).tobytes() == b[1].astype(np.float32).tobytes(), (what, "scores")
    assert a[2].tolist() == b[2].tolist(), (what, "counts")


def _against_exact(g, qs, radii, cap, order, fn="range_batch_device", host_every=8):
    """the batch on the route and under mode 0: bit-equal; every host_every-th query with a radius the host API takes against
    VecSimIndex_RangeQuery.  Returns the route's (labels, scores, counts, path, flags)."""
    got = _run(g, qs, radii, cap, order, 1, fn)
    want = _run(g, qs, radii, cap, order, 0, fn)
    assert want[3] == 0 and (want[4] == 0).all()
    _same(got, want, (fn, order, cap))
    if host_every and fn == "range_batch_device":
        for i in range(0, qs.shape[0], host_every):
            r = float(radii[i])
            if not r >= 0:
                continue
            ei, es, code = g.range(qs[i], r, order)
            assert code == 0 and int(got[2][i]) == len(ei), (i, r)
            if len(ei) <= cap:
                assert got[0][i, :len(ei)].tolist() == ei.tolist(), i
                assert got[1][i, :len(ei)].astype(np.float32).tobytes() == es.astype(np.float32).tobytes(), i
    return got


def _exact_topk(g, qs, k):
    """(labels, scores) of the exact scan's top-k (mode 0): the CUDA-core distances"""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(0)
    try:
        lab, sc, rc = g.topk_batch(qs, k)
    finally:
        vs.lib().VecSimB200_SetCoarseMode(1)
    assert rc == 0
    return lab.astype(np.int64), sc.astype(np.float32)


def _radii_at(g, qs, ranks):
    _, sc = _exact_topk(g, qs, max(ranks))
    return np.array([sc[i, ranks[i % len(ranks)] - 1] for i in range(qs.shape[0])], dtype=np.float32)


def _queries(vtype, metric, seed, nq, dim):
    qs = ol.synth_rows(vtype, seed, 0, nq, dim)
    if metric == ol.IP:  # 1 - dot mostly positive: the host API takes the radii too
        qs = to16(decode16(qs, vtype) / math.sqrt(dim), vtype)
    return qs


# ------------------------------------------------------------------------------------------------------------------
# GPU: the route against the exact scan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.COS])
@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_route_equals_the_exact_scan(mode1, vtype, metric):
    n = 70_000
    for dim in (32, 128, 768, WGMMA_MAX_DIM):
        rows = ol.synth_rows(vtype, 100 + dim, 0, n, dim)
        rows[3000:3010] = rows[100]  # ties: ten copies of one row
        g = _index(vtype, metric, dim, rows)
        qs = _queries(vtype, metric, 200 + dim, 256, dim)
        qs[1] = rows[100]
        radii = _radii_at(g, qs, [1, 10, 100, 1000])
        for nq in (16, 40, 256):
            for cap, order in ((512, BY_SCORE), (4096, BY_ID)):
                got = _against_exact(g, qs[:nq], radii[:nq], cap, order, host_every=8 if nq == 40 else 0)
                assert got[3] == 2 and got[4].tolist() == [1] * nq, (dim, nq, got[3], got[4][:8])
                if cap == 512:
                    assert (got[2][3::4] > 512).any()  # the 1000th-neighbour radii overflow this cap: padded rows
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.COS])
@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_margin_at_work(mode1, vtype, metric):
    """tc scores from the direct KNN route (mode 1), cc scores from the exact scan (mode 0).  A radius equal to the cc score of a
    row whose tc is above it keeps that row; a radius one float below the cc score of a row whose tc is below it drops it.  The
    largest |tc - cc| / eps16_q over the returned rows is printed and must be at most 1."""
    from test_half_precision_bounds import device_batch

    n, dim, nq, k = 70_000, 256, 64, 128
    rows = ol.synth_rows(vtype, 301, 0, n, dim)
    g = _index(vtype, metric, dim, rows)
    qs = _queries(vtype, metric, 302, nq, dim)
    st = _stored(g, qs)
    tl, ts = device_batch(g, st[:, :2 * dim].copy().view(np.uint16), k)
    assert _vs().lib().VecSimB200_LastBatchPath(g.h) == 2
    cl, cs = _exact_topk(g, qs, k)
    out = np.empty((n, dim), dtype=np.uint16)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, out.ctypes.data) == 0
    X = decode16(out, vtype)
    max_norm = np.float32(np.sqrt(np.max(np.einsum("ij,ij->i", X, X))))
    radii = np.zeros(nq, dtype=np.float32)
    probe = np.full(nq, -1, dtype=np.int64)
    inside = np.zeros(nq, dtype=bool)
    worst = 0.0
    for i in range(nq):
        cc = dict(zip(cl[i].tolist(), cs[i].tolist()))
        qn = float(np.sqrt(np.sum(decode16(st[i, :2 * dim].view(np.uint16), vtype) ** 2)))
        e16, _ = eps16(dim, max_norm, qn)
        both = [(lab, float(t), cc[lab]) for lab, t in zip(tl[i].tolist(), ts[i].tolist()) if lab in cc]
        worst = max([worst] + [abs(t - c) / e16 for _, t, c in both])
        want_above = i % 2 == 0
        pick = [(lab, c) for lab, t, c in both if (np.float32(t) > np.float32(c)) == want_above and np.float32(t) != np.float32(c)]
        if pick:
            lab, c = pick[len(pick) // 2]
            probe[i], inside[i] = lab, want_above
            radii[i] = np.float32(c) if want_above else np.nextafter(np.float32(c), np.float32(-np.inf))
        else:
            radii[i] = cs[i, 9]
    assert (probe >= 0).sum() >= nq // 4, "too few rows whose tensor-core score differs from the exact one"
    got = _against_exact(g, qs, radii, 1024, BY_SCORE)
    assert got[3] == 2 and (got[4] == 1).all(), got[4]
    for i in np.flatnonzero(probe >= 0):
        members = got[0][i, :int(got[2][i])].tolist()
        assert (probe[i] in members) == inside[i], (i, probe[i], inside[i])
    print(f"\n[|tc - cc| / eps16] {'fp16' if vtype == ol.F16 else 'bf16'} {'IP' if metric == ol.IP else 'COS'}: "
          f"{worst:.4g} ({int((probe >= 0).sum())} probes)")
    assert worst <= 1.0
    g.close()


# ------------------------------------------------------------------------------------------------------------------
# GPU: dynamic range, edge radii, queries and rows outside the route
# ------------------------------------------------------------------------------------------------------------------
def _fp16_with_subnormals(rng, n, dim, frac):
    x = rng.uniform(-1, 1, (n, dim)).astype(np.float16)
    sub = rng.random((n, dim)) < frac
    x[sub] = (rng.integers(1, 1024, int(sub.sum())) * np.where(rng.random(int(sub.sum())) < 0.5, -1, 1)).astype(np.float64) * 2.0 ** -24
    return x.view(np.uint16)


@pytest.mark.gpu
def test_fp16_subnormals_and_largest_values(mode1):
    rng = np.random.default_rng(11)
    n, dim, nq = 70_000, 128, 40
    rows = _fp16_with_subnormals(rng, n, dim, 0.5)
    rows[1000:3000] = _fp16_with_subnormals(rng, 2000, dim, 1.0)
    rows[5000:5050, :4] = np.float16(65504.0).view(np.uint16)
    qs = _fp16_with_subnormals(rng, nq, dim, 0.5)
    qs[:8] = _fp16_with_subnormals(rng, 8, dim, 1.0)
    g = _index(ol.F16, ol.IP, dim, rows)
    radii = _radii_at(g, qs, [1, 10, 100])
    got = _against_exact(g, qs, radii, 1024, BY_SCORE, host_every=3)
    assert got[3] == 2


@pytest.mark.gpu
def test_bf16_subnormal_products(mode1):
    """bf16 rows near 1e-20 and queries near 1e-19 in half of the dimensions: every product there lies in the fp32 subnormal
    range, while the other half spreads the distances"""
    n, dim, nq = 70_000, 64, 16
    rows = decode16(ol.synth_rows(ol.BF16, 21, 0, n, dim), ol.BF16)
    rows[:, 32:] *= 1e-20
    qs = decode16(_queries(ol.BF16, ol.IP, 23, nq, dim), ol.BF16)
    qs[:, 32:] *= 1e-19
    rows, qs = to16(rows, ol.BF16), to16(qs, ol.BF16)
    g = _index(ol.BF16, ol.IP, dim, rows)
    radii = _radii_at(g, qs, [1, 10, 100])
    got = _against_exact(g, qs, radii, 4096, BY_ID, host_every=1)
    assert got[3] == 2 and (got[4] == 1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_edge_radii_and_non_finite_queries(mode1, vtype):
    """+-0, NaN, +inf and negative radii; queries with an inf or NaN component take the exact scan while the rest stay on the route"""
    n, dim, nq = 70_000, 64, 24
    rows = ol.synth_rows(vtype, 31, 0, n, dim)
    g = _index(vtype, ol.IP, dim, rows)
    qs = _queries(vtype, ol.IP, 32, nq, dim)
    _, cs = _exact_topk(g, qs, 100)
    radii = cs[:, 30].copy()  # the 31st neighbour: 1 - dot below zero
    radii[0], radii[1], radii[2], radii[3] = 0.0, -0.0, np.nan, np.inf
    radii[4], radii[5] = cs[4, 0], np.nextafter(cs[5, 0], np.float32(-np.inf))  # at the best row, one float below it
    inf16, nan16 = to16(np.array([np.inf, np.nan], dtype=np.float32), vtype)
    qs[6, 3], qs[7, 0] = inf16, nan16
    for order in (BY_SCORE, BY_ID):
        got = _against_exact(g, qs, radii, 4096, order, host_every=1)
        assert got[3] == 2
        f = got[4]
        assert f[2] == 0 and f[3] == 0 and f[6] == 0 and f[7] == 0, f
        assert (np.delete(f, [2, 3, 6, 7]) == 1).all(), f
        assert got[2][2] == 0 and got[2][3] == n and got[2][5] == 0 and got[2][4] >= 1
        assert (radii[8:] < 0).sum() >= 8  # negative radii on the route


@pytest.mark.gpu
def test_bf16_row_norm_overflowing_float_leaves_the_route(mode1):
    n, dim, nq = 70_000, 64, 16
    rows = ol.synth_rows(ol.BF16, 41, 0, n, dim)
    rows[777] = to16(np.full((1, dim), 1e20, dtype=np.float32), ol.BF16)[0]  # |row|^2 = 6.4e41: inf in fp32
    g = _index(ol.BF16, ol.IP, dim, rows)
    qs = _queries(ol.BF16, ol.IP, 42, nq, dim)
    radii = _radii_at(g, qs, [10])
    got = _against_exact(g, qs, radii, 1024, BY_SCORE)
    assert got[3] == 0 and (got[4] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_clustered_lists_overflow_to_the_exact_scan(mode1, vtype):
    """40,000 near-copies of one row stored together: a query at that row with a radius reaching them overflows its lists (flag 0,
    the exact scan's answer); the others keep flag 1"""
    n, dim, nq = 70_000, 128, 16
    rows = ol.synth_rows(vtype, 51, 0, n, dim)
    base = decode16(rows[10], vtype)
    near = base[None, :] * (1.0 + 1e-3 * np.random.default_rng(5).standard_normal((40_000, 1)))
    rows[20_000:60_000] = to16(near, vtype)
    g = _index(vtype, ol.IP, dim, rows)
    qs = _queries(vtype, ol.IP, 52, nq, dim)
    qs[3] = rows[10]
    radii = _radii_at(g, qs, [10])
    _, cs = _exact_topk(g, qs[3:4], 1)
    radii[3] = np.float32(cs[0, 0] + 0.5 * abs(cs[0, 0]) + 0.5)
    for order in (BY_SCORE, BY_ID):
        got = _against_exact(g, qs, radii, 1024, order)
        assert got[3] == 2 and got[4][3] == 0 and got[4].sum() == nq - 1, got[4]
        assert got[2][3] >= 40_000 and (got[0][3] == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.F16, ol.BF16])
def test_mutations_between_batches(mode1, vtype):
    """an appended row of a much larger norm (X must rise), an in-place overwrite, a swap-delete followed by id reuse: each batch
    after them equals the exact scan"""
    n, dim, nq = 70_000, 128, 16
    rows = ol.synth_rows(vtype, 61, 0, n, dim)
    g = _index(vtype, ol.IP, dim, rows)
    qs = _queries(vtype, ol.IP, 62, nq, dim)
    radii = _radii_at(g, qs, [10])
    assert _against_exact(g, qs, radii, 256, BY_SCORE)[3] == 2
    big = to16(decode16(qs[0:1], vtype) * 200.0, vtype)  # |row| ~ 200 |q| sqrt(dim): far inside every radius of query 0
    assert g.add_many(big, label0=n + 1) == 1
    got = _against_exact(g, qs, radii, 256, BY_SCORE)
    assert got[3] == 2 and n + 1 in got[0][0, :int(got[2][0])].tolist()
    for i in range(0, nq, 2):
        g.add(qs[i], 5 + i)  # overwrite in place with the query itself
    got = _against_exact(g, qs, radii, 256, BY_ID)
    assert got[3] == 2
    for lab in (8, 9_000, 40_001):
        g.delete(lab)
    assert g.add_many(ol.synth_rows(vtype, 63, 0, 3, dim), label0=n + 10) == 3  # the freed ids are reused
    for order in (BY_SCORE, BY_ID):
        got = _against_exact(g, qs, radii, 256, order)
        assert got[3] == 2 and (got[4] == 1).all()


# ------------------------------------------------------------------------------------------------------------------
# GPU: multi-value indexes, shard groups, the caller's stream
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_multi_value_label_range(mode1):
    """3 rows per label: the route's rows are folded per label (flag 1); a query with more than 4,096 hit rows gets flag 3 and
    the exact fold's answer"""
    n, dim, nq = 70_002, 128, 16
    rows = ol.synth_rows(ol.F16, 71, 0, n, dim)
    labels = (np.arange(n) // 3 + 1).astype(np.uint64)
    g = _index(ol.F16, ol.IP, dim, rows, labels=labels, multi=True)
    qs = _queries(ol.F16, ol.IP, 72, nq, dim)
    _, cs = _exact_topk(g, qs, 100)
    radii = cs[:, 50].copy()
    single = _index(ol.F16, ol.IP, dim, rows)
    _, rs = _exact_topk(single, qs[:1], 6000)
    radii[0] = rs[0, 5000]  # 5,001 hit rows
    single.close()
    for order in (BY_SCORE, BY_ID):
        got = _against_exact(g, qs, radii, 4096, order, fn="label_range_batch_device")
        assert got[3] == 2 and got[4][0] == 3 and (got[4][1:] == 1).all(), got[4]


@pytest.mark.gpu
def test_shard_group_of_one_is_the_local_call(mode1):
    import torch

    L = mode1.lib()
    n, dim, nq, cap = 70_000, 128, 16, 512
    rows = ol.synth_rows(ol.BF16, 81, 0, n, dim)
    g = _index(ol.BF16, ol.COS, dim, rows)
    qs = _queries(ol.BF16, ol.COS, 82, nq, dim)
    radii = _radii_at(g, qs, [20])
    local = _run(g, qs, radii, cap, BY_SCORE)
    assert local[3] == 2 and (local[4] == 1).all()
    grp = L.VecSimB200_ShardGroup_New(None, 0, 1)
    assert grp
    try:
        s = _stream()
        with torch.cuda.stream(s):
            qd = torch.from_numpy(_stored(g, qs)).cuda()
            rd = torch.from_numpy(radii).cuda()
            lab = torch.empty((nq, cap), dtype=torch.int64, device="cuda")
            sc = torch.empty((nq, cap), dtype=torch.float32, device="cuda")
            cnt = torch.empty(nq, dtype=torch.int32, device="cuda")
            rc = L.VecSimB200_ShardGroup_RangeQueryBatchDevice(grp, g.h, qd.data_ptr(), nq, rd.data_ptr(), cap, BY_SCORE, lab.data_ptr(),
                                                               sc.data_ptr(), cnt.data_ptr(), C.c_void_p(s.cuda_stream))
        s.synchronize()
        assert rc == 0
        _same((lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), local, "world = 1")
        assert L.VecSimB200_LastBatchPath(g.h) == 2
    finally:
        L.VecSimB200_ShardGroup_Free(grp)


@pytest.mark.gpu
def test_outputs_feed_torch_on_the_callers_stream(mode1):
    import torch

    n, dim, nq = 70_000, 128, 64
    rows = ol.synth_rows(ol.F16, 91, 0, n, dim)
    g = _index(ol.F16, ol.COS, dim, rows)
    qs = ol.synth_rows(ol.F16, 92, 0, nq, dim)
    radii = _radii_at(g, qs, [10])
    d_q = torch.from_numpy(_stored(g, qs)).cuda()
    d_r = torch.from_numpy(radii).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        lab, sc, cnt, rc = g.range_batch_device(d_q, d_r, 64, BY_SCORE, stream=s)
        hits = (lab >= 0).sum(dim=1).to(torch.int32)  # consumed on the same stream, no host sync in between
        total = cnt.sum()
    s.synchronize()
    assert rc == 0 and mode1.lib().VecSimB200_LastBatchPath(g.h) == 2
    assert hits.cpu().tolist() == cnt.cpu().tolist()
    assert int(total.item()) >= 10 * nq
