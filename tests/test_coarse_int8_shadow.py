"""The int8 copy of unit fp32 rows (cosine batches with k <= 128, DESIGN.md §4.2): the approximate pass runs on int8 operands with
one scale per 128-row tile and a per-query error bound; rescoring stays in fp32, so labels and score bits must equal the exact
scan's whatever tier answers.

The first test is CPU-only: a numpy restatement of the quantization and of the bound of quantize_queries_kernel, checked in
fp64 on rows and queries built to make the rounding errors add up.  The others run on the GPU against the exact scan of the
same index (coarse mode 0), which the rest of the suite holds to the reference bit for bit.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

import oracle_lib as ol

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "redisearch_b200", "csrc")


def _quant(x, axis_max):
    """int8 quantization as the kernels do it: s = max|x| / 127 in fp32 (1 for zero), rint(x / s) clamped to +-127."""
    x = np.asarray(x, dtype=np.float32)
    m = np.float32(axis_max)
    s = np.float32(m / np.float32(127.0)) if m > 0 else np.float32(1.0)
    q = np.clip(np.rint(x / s), -127, 127)
    return s, q


def _eps(q, eta_n, delta_max, x_max, dim):
    """quantize_queries_kernel's bound, in fp64."""
    qn = float(np.linalg.norm(q.astype(np.float64)))
    e = qn * delta_max + eta_n * x_max + eta_n * delta_max + (dim + 8) * 2.0 ** -23 * (qn + eta_n) * (x_max + delta_max) + 2.0 ** -21
    return e * 1.0001


def _midpoint_rows(rng, n, dim, signs=None):
    """Unit rows whose elements sit at (m + 1/2) s of the scale s that every row of the set shares (one element at 127 s in every
    row, the same magnitudes permuted): each rounds at a midpoint.  signs (optional [dim]): the sign pattern of every row."""
    mags = rng.integers(0, 126, size=dim).astype(np.float64) + 0.5
    mags[0] = 127.0
    mags /= np.linalg.norm(mags)
    out = np.empty((n, dim), dtype=np.float32)
    for i in range(n):
        v = rng.permutation(mags)
        sg = signs if signs is not None else rng.choice([-1.0, 1.0], size=dim)
        out[i] = (v * sg).astype(np.float32)
    return out


def _aligned_query(rng, x, s_t, qx):
    """A unit query at int8 midpoints whose signs follow the row's residual (q . delta > 0) and whose own residual follows the
    row (eta . x > 0): all three error terms of the bound point the same way."""
    dim = x.shape[0]
    delta = x.astype(np.float64) - float(s_t) * qx
    sg = np.where(delta >= 0, 1.0, -1.0)
    n = rng.integers(0, 60, size=dim) * 2  # even: rint of n + 1/2 rounds down, eta = +s/2 in the magnitude's direction
    n = np.where(np.sign(x) == sg, n, n + 1)  # odd: rounds up, eta = -s/2 in the magnitude's direction
    v = (n + 0.5) * sg
    v[0] = 127.0 * np.sign(v[0]) if v[0] != 0 else 127.0
    return (v / np.linalg.norm(v)).astype(np.float32)


# The restatement above rests on these lines of coarse_tc.cu: the scale, rounding and clamp of rows and queries, the running maxima
# rounded up, the bound of quantize_queries_kernel and the 2 eps of threshold_kernel's T and of refine_kernel's cut
_PINNED = (
    "const float sc = m > 0.0f ? __fdiv_rn(m, 127.0f) : 1.0f;",
    "const float qv = fminf(fmaxf(rintf(__fdiv_rn(f[h], sc)), -127.0f), 127.0f);",
    "const float rn = __double2float_ru(sqrt(res2));",
    "w_nrm = fmaxf(w_nrm, __double2float_ru(sqrt(nrm2)));",
    "const float sc = (finite && m > 0.0f) ? __fdiv_rn(m, 127.0f) : 1.0f;",
    "const float qv = fminf(fmaxf(rintf(__fdiv_rn(v, sc)), -127.0f), 127.0f);",
    "double e = qn * D + en * X + en * D + (double)(dim + 8) * 0x1p-23 * (qn + en) * (X + D) + 0x1p-21;",
    "e *= 1.0001;",
    "const float ef = __double2float_ru(e);",
    "T = key_to_float(ak) + (2.0f * e) * 1.001f + 1e-30f;",
    "key_to_float(ak_key) + (2.0f * eps) * 1.001f + 1e-30f;",
)


def test_int8_restatement_is_pinned_to_the_kernels():
    with open(os.path.join(CSRC, "coarse_tc.cu")) as f:
        src = f.read()
    for line in _PINNED:
        assert line in src, line


def _f32_up(v):
    """__double2float_ru of a non-negative double."""
    f = np.float32(v)
    return float(np.nextafter(f, np.float32(np.inf))) if float(f) < v else float(f)


def _stored(x):
    """normalize_f32 (csrc/host_numeric.h) row by row: what a cosine index stores."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    norm = np.sqrt((x.astype(np.float64) ** 2).sum(axis=1)).astype(np.float32)
    return (x / norm[:, None]).astype(np.float32)


def _corpus_stats(rows):
    """to_i8_tiled_kernel over rows [0, n) from tile 0: (delta_max, x_max), each row's residual and norm rounded up."""
    rows = np.asarray(rows, dtype=np.float32)
    dmax = xmax = 0.0
    for t0 in range(0, rows.shape[0], 128):
        tile = rows[t0:t0 + 128]
        s, q = _quant(tile, np.abs(tile).max())
        res = np.sqrt(((tile.astype(np.float64) - float(s) * q) ** 2).sum(axis=1)).max()
        nrm = np.sqrt((tile.astype(np.float64) ** 2).sum(axis=1)).max()
        dmax, xmax = max(dmax, _f32_up(res)), max(xmax, _f32_up(nrm))
    return dmax, xmax


def _query_eps(q, delta_max, x_max):
    """quantize_queries_kernel for one stored query: (s_q, q~, eps_q)."""
    s_q, qq = _quant(q, np.abs(q).max())
    eta_n = float(np.linalg.norm(q.astype(np.float64) - float(s_q) * qq))
    return s_q, qq, _f32_up(_eps(q, eta_n, delta_max, x_max, q.shape[0]))


def _approx(rows, q, s_q, key=False):
    """s_q s_t q~.x~ of every row in fp64, each row quantized with the scale of its 128-row tile (rows [0, n) from tile 0); key:
    also the distance the kernel computes in fp32, 1 - fl(fl(s_q s_t) acc)."""
    rows = np.asarray(rows, dtype=np.float32)
    _, qq = _quant(q, np.abs(q).max())
    out, d32 = np.empty(rows.shape[0]), np.empty(rows.shape[0], dtype=np.float32)
    for t0 in range(0, rows.shape[0], 128):
        tile = rows[t0:t0 + 128]
        s_t, xt = _quant(tile, np.abs(tile).max())
        acc = xt.astype(np.int64) @ qq.astype(np.int64)
        assert np.abs(acc).max() < 2 ** 24
        out[t0:t0 + 128] = float(s_q) * float(s_t) * acc
        d32[t0:t0 + 128] = np.float32(1.0) - np.float32(s_q * s_t) * acc.astype(np.float32)
    return (out, d32) if key else out


SPIKE = np.float32(0.3)  # sets the scale of every tile holding planted rows: s_t = fl(0.3 / 127)
TAU = 2.0 ** -12         # distance of a planted component from its rounding midpoint, in units of s_t


def flat_query(rng, dim):
    """Family (a): q = sign pattern / sqrt(dim).  Every component quantizes to +-127 exactly: eta ~ 0, eps_q ~ delta_max."""
    return _stored(np.where(rng.random(dim) < 0.5, -1.0, 1.0).astype(np.float32))[0]


def spiky_query(rng, dim, spike=0.6):
    """Family (b): one component at 127 s_q, every other one TAU s_q off an int8 midpoint (n + 1/2) s_q, on a random side:
    |eta| ~ s_q sqrt(dim) / 2, so that the |eta| x_max term is about twice |q| delta_max."""
    s = spike / 127.0
    g = np.abs(rng.standard_normal(dim))
    g *= math.sqrt(1.0 - spike * spike) / np.linalg.norm(g)
    v = (np.floor(g / s) + 0.5 + np.where(rng.random(dim) < 0.5, -TAU, TAU)) * s
    v[int(rng.integers(dim))] = 127.0 * s
    v *= np.where(rng.random(dim) < 0.5, -1.0, 1.0)
    return _stored((v / np.linalg.norm(v)).astype(np.float32))[0]


def planted_rows(q, nb, margin=(2e-4, 1e-3)):
    """Row A and nb rows B for the stored query q, unit rows that all quantize with one tile scale s_t = fl(SPIKE / 127): one
    component is the spike (the query's own spike, or for a flat query any), one absorbs the norm (the smallest |q_i|), and every other sits TAU s_t
    off a rounding midpoint (m + 1/2) s_t.  A sits on the side that rounds its residual delta along q (q.delta_A ~ +|delta|), the B
    rows on the other (q.delta_B ~ -|delta|).  A flat query (family a) aims every row at q.  A spiky query (family b) aims A and B
    along q with +-0.53 of their norm along eta (orthogonalised against q), so that the eta.x term pushes A back and B forward at
    equal q.x.  B rows differ by one grid step on one component of the largest |q_i|; A takes whole grid steps on its components with the largest |q_i|
    until it beats every B in exact arithmetic by a margin within `margin`.  Returns (A [dim], B [nb, dim]) as a cosine index
    stores them."""
    q64 = q.astype(np.float64)
    dim = q.shape[0]
    s_q, qq = _quant(q, np.abs(q).max())
    eta = q64 - float(s_q) * qq
    order = np.argsort(np.abs(q64), kind="stable")
    flat = np.linalg.norm(eta) < 1e-3
    # spike: on the query's own spike where it has one (no other component of the row may outgrow it), slack: the smallest |q_i|
    js, jl = (int(order[1]), int(order[0])) if flat else (int(order[-1]), int(order[0]))
    free = np.ones(dim, dtype=bool)
    free[[js, jl]] = False
    sg = np.where(q64 < 0, -1.0, 1.0)
    st = float(np.float32(SPIKE / np.float32(127.0)))
    qf = np.where(free, q64, 0.0)
    qf /= np.linalg.norm(qf)
    e = np.where(free, eta, 0.0)
    e -= (e @ qf) * qf
    c, g = (1.0, 0.0) if flat else (0.85, math.sqrt(1 - 0.85 ** 2))
    if not flat:
        e /= np.linalg.norm(e)

    def base(d, against):  # grid indices m and midpoint sides of the direction d, scaled so that the slack stays in (0.05, 0.25)
        r = math.sqrt(1.0 - float(SPIKE) ** 2 - 0.15 ** 2)
        for _ in range(400):
            t = d * r
            m = np.floor(np.abs(t) / st)
            sx = np.where(t != 0, np.sign(t), sg)
            mag = (m + 0.5) * st
            rest = 1.0 - float(SPIKE) ** 2 - float((mag[free] ** 2).sum())
            if 0.05 ** 2 <= rest <= 0.25 ** 2:
                break
            r *= 0.999 if rest < 0.05 ** 2 else 1.001
        below = (sx == sg) if against else (sx != sg)  # just below a midpoint: rounds toward zero, delta signed like x
        return m, sx, np.where(below, -TAU, TAU)

    def row(m, sx, off):
        v = sx * (m + 0.5 + off) * st
        v[js], v[jl] = sg[js] * float(SPIKE), 0.0
        rest = 1.0 - float((v ** 2).sum())
        assert 0.0 < rest < 0.25 ** 2, rest
        v[jl] = sg[jl] * math.sqrt(rest)
        return _stored(v.astype(np.float32))[0]

    ma, sxa, offa = base(c * qf + g * e, True)
    mb, sxb, offb = base(c * qf - g * e, False)
    steps = [int(j) for j in np.argsort(-np.abs(np.where(free, q64, 0.0)), kind="stable") if np.abs(q64[j]) < 2.0 / math.sqrt(dim)]
    assert nb <= len(steps)
    bs = []
    for i in range(nb):
        m = mb.copy()
        m[steps[i]] += 1.0  # distinct B rows
        bs.append(row(m, sxb, offb))
    b = np.stack(bs)
    best_b = float((b.astype(np.float64) @ q64).max())
    m = ma.copy()
    for j in steps:
        a = row(m, sxa, offa)
        gap = float(a.astype(np.float64) @ q64) - best_b
        if margin[0] <= gap <= margin[1]:
            break
        up = (gap < margin[0]) == (sxa[j] == sg[j])  # one grid step towards q (or away from it)
        if up or m[j] > 0:
            m[j] += 1.0 if up else -1.0
    assert margin[0] <= gap <= margin[1], gap
    return a, b


def test_int8_bound_covers_worst_case_rounding():
    """|approx - exact| <= eps_q in fp64 for rows and queries at rounding midpoints with aligned signs, and the distance the kernel
    computes in fp32, 1 - fl(fl(s_q s_t) acc), stays within eps_q of the fp64 distance.
    Then the planted construction (planted_rows): on the rows the index stores, in their own tiles after Gaussian filler, A stays
    within eps_q and rounds within 5 % of it against the query, the B rows within 5 % of it with the query, so the int8 pass puts
    A at least 1.9 eps_q behind the k-th B for a flat query (family a): the refine cut a_k + 2 eps_q reaches A with nothing to
    spare, and a bound 5 % short drops it.  A spiky query (family b) has an eps_q at least three times as large, and its rows
    reach 1.0 eps_q (1.05 measured), half of it from the eta.x term: a bound without the |eta| x_max term (a third of eps_q)
    drops A."""
    rng = np.random.default_rng(7)
    for dim in (64, 384, 520, 768, 1024):
        tile = _midpoint_rows(rng, 128, dim)
        s_t, qt = _quant(tile, np.abs(tile).max())
        res = np.linalg.norm(tile.astype(np.float64) - float(s_t) * qt, axis=1)
        delta_max = float(np.float32(res.max()) * np.float32(1 + 2 ** -20))
        x_max = float(np.linalg.norm(tile.astype(np.float64), axis=1).max())
        for r in range(0, 128, 16):
            q = _aligned_query(rng, tile[r], s_t, qt[r])
            s_q, qq = _quant(q, np.abs(q).max())
            eta_n = float(np.linalg.norm(q.astype(np.float64) - float(s_q) * qq))
            eps = _eps(q, eta_n, delta_max, x_max, dim)
            for j in range(128):
                exact = float(q.astype(np.float64) @ tile[j].astype(np.float64))
                acc = int(qq.astype(np.int64) @ qt[j].astype(np.int64))
                assert abs(acc) < 2 ** 24  # exact in float
                approx64 = float(s_q) * float(s_t) * acc
                assert abs(approx64 - exact) <= eps
                d32 = np.float32(1.0) - np.float32(np.float32(s_q * s_t) * np.float32(acc))
                assert abs(float(d32) - (1.0 - exact)) <= eps
    k = 128
    for dim in (256, 520, 768, 1024):
        filler = _stored(rng.standard_normal((512, dim)).astype(np.float32))
        for family in ("a", "b"):
            q = flat_query(rng, dim) if family == "a" else spiky_query(rng, dim)
            a, b = planted_rows(q, k + 1)
            tiles = [np.concatenate([a[None], b[:127]]), np.concatenate([b[127:], filler[: 128 - (k + 1 - 127)]])]
            corpus = np.concatenate([filler] + tiles)
            delta_max, x_max = _corpus_stats(corpus)
            s_q, qq, eps = _query_eps(q, delta_max, x_max)
            q64 = q.astype(np.float64)
            exact = corpus.astype(np.float64) @ q64
            approx, d32 = _approx(corpus, q, s_q, key=True)
            assert (np.abs(approx - exact) <= eps).all()
            assert (np.abs(d32.astype(np.float64) - (1.0 - exact)) <= eps).all()
            ia, ib = 512, np.r_[513:640, 640:642]
            assert exact[ia] > exact[ib].max()  # A is in the exact top-k
            err_a, err_b = exact[ia] - approx[ia], approx[ib] - exact[ib]
            power = (1.0 - approx[ia]) - np.sort(1.0 - approx[ib])[k - 1]
            if family == "a":
                assert err_a >= 0.95 * eps and err_b.min() >= 0.95 * eps, (dim, err_a / eps, err_b.min() / eps)
                assert power >= 1.9 * eps, (dim, power / eps)
            else:
                eps_a = _query_eps(flat_query(rng, dim), delta_max, x_max)[2]
                assert eps >= 3.0 * eps_a, (dim, eps / eps_a)
                assert power >= 1.0 * eps, (dim, power / eps)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------------
def _device_batch(vs, torch, index, qn, k):
    nq = qn.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qn)).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert vs.lib().VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)  # -1 after the exact scan alone
    return out_l.cpu().numpy(), out_s.cpu().numpy(), (flags if frc == 0 else None)


def _normalized(qs):
    qn = qs.astype(np.float32).copy()
    for i in range(qn.shape[0]):
        ol.port().orc_normalize(ol._p(qn[i]), qn.shape[1], ol.F32)
    return qn


def _check_against_exact(vs, torch, g, qs, k, bits=8):
    """The batch on the int8 copy (asserted) against the exact scan of the same index: labels and score bits equal."""
    qn = _normalized(qs)
    vs.lib().VecSimB200_SetCoarseMode(1)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    assert vs.lib().VecSimB200_LastCoarseShadowBits(g.h) == bits
    vs.lib().VecSimB200_SetCoarseMode(0)
    el, es, _ = _device_batch(vs, torch, g, qn, k)
    vs.lib().VecSimB200_SetCoarseMode(-1)
    for i in range(qs.shape[0]):
        assert labels[i].tolist() == el[i].tolist(), (i, flags[i], labels[i], el[i])
        assert scores[i].tobytes() == es[i].tobytes(), (i, flags[i])
    return flags


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nq,k", [(256, 256, 10), (384, 17, 1), (520, 200, 10), (768, 16, 128), (1024, 256, 10), (768, 256, 10),
                                      (384, 200, 128), (1024, 17, 1)])
def test_int8_route_is_exact(dim, nq, k):
    import torch

    from redisearch_b200 import vecsim as vs

    n = 65_536 + 300
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags != 0).sum() >= nq * 0.9, flags
    # the host-facing batch entry point goes through the same pipeline; a single query rides the copy the batch built
    hl, hs, rc = g.topk_batch(qs[:4], k)
    assert rc == 0
    vs.lib().VecSimB200_SetCoarseMode(1)
    for i in range(2):
        gi, gs, code = g.topk(qs[i], k)
        assert code == 0 and gi.tolist() == hl[i].astype(np.int64).tolist()
        assert vs.lib().VecSimB200_LastCoarseShadowBits(g.h) == 8
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
def test_int8_route_is_exact_at_rounding_midpoints_and_near_ties():
    """Rows at int8 rounding midpoints whose signs follow the queries', near-duplicates one ulp apart at the k-th distance: the
    answer stays exact (tiers may fall back)."""
    import torch

    from redisearch_b200 import vecsim as vs

    rng = np.random.default_rng(11)
    dim, nq, k = 384, 24, 10
    filler = ol.synth_rows(ol.F32, 42, 0, 516 * 128, dim)  # whole tiles: every crafted block below is a tile of its own
    filler /= np.linalg.norm(filler, axis=1, keepdims=True)
    qs = _midpoint_rows(rng, nq, dim)
    blocks = [filler]
    for i in range(nq):  # one tile per query, rows with its sign pattern: they score high against it, share the tile's scale
        blocks.append(_midpoint_rows(rng, 128, dim, signs=np.sign(qs[i])))  # and so round at its midpoints
    near = []
    for i in range(nq):  # near-ties, in tiles after the crafted ones: copies of a close row with one element moved by an ulp
        base = blocks[1 + i][0]
        for t in range(12):
            r = base.copy()
            j = rng.integers(0, dim)
            r[j] = np.nextafter(r[j], np.float32(np.inf if t % 2 else -np.inf))
            near.append(r)
    blocks.append(np.asarray(near, dtype=np.float32))
    rows = np.ascontiguousarray(np.concatenate(blocks).astype(np.float32))
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == rows.shape[0]
    _check_against_exact(vs, torch, g, qs, k)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [64, 128])
def test_narrow_rows_keep_the_fp16_copy(dim):
    """Up to 128 dimensions an int8 row is padded to as many bytes as the fp16 row: those batches keep the fp16 copy."""
    import torch

    from redisearch_b200 import vecsim as vs

    n, nq, k = 66_000, 32, 10
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(ol.synth_rows(ol.F32, 42, 0, n, dim), label0=1) == n
    _check_against_exact(vs, torch, g, ol.synth_rows(ol.F32, 43, 0, nq, dim), k, bits=16)


@pytest.mark.gpu
def test_single_queries_ride_the_copy_their_route_reads():
    """A single query takes a tensor-core route only when the copy that route reads is current.  KNN queries read the int8 copy
    a KNN batch built, and a mutation sends them to the exact scan until the next batch.  Small range batches read the fp16
    copy: after KNN batches alone they take the exact scan and build nothing, and once a large range batch has built the fp16
    copy they ride it, with the int8 copy kept as it was."""
    import torch

    from redisearch_b200 import vecsim as vs

    n, dim, k = 70_000, 384, 10
    rows = ol.synth_rows(ol.F32, 42, 0, n + 1, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows[:n], label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, 20, dim)
    vs.lib().VecSimB200_SetCoarseMode(1)

    def single(expect_path, expect_bits):
        for q in qs[:3]:
            _, _, code = g.topk(q, k)
            assert code == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == expect_path
            if expect_path:
                assert vs.lib().VecSimB200_LastCoarseShadowBits(g.h) == expect_bits

    def small_range(expect_flag):
        replies, rc, flags = g.range_batch(qs[:4], 0.9)
        assert rc == 0 and (flags == expect_flag).all(), flags
        return [r[0].tolist() for r in replies]

    single(0, 0)  # no copy yet
    _check_against_exact(vs, torch, g, qs, k)  # a KNN batch builds the int8 copy
    vs.lib().VecSimB200_SetCoarseMode(1)
    single(1, 8)
    before = small_range(0)  # no fp16 copy: the exact scan, and none is built
    single(1, 8)
    _, rc, flags = g.range_batch(qs[:16], 0.9)  # a batch of 16 builds the fp16 copy
    assert rc == 0 and (flags == 1).all()
    assert small_range(1) == before  # now small range batches ride it
    single(1, 8)  # the int8 copy is still current
    assert g.add(rows[n], n + 1) == 1  # stale copies: single queries do not pay for the refresh
    single(0, 0)
    small_range(0)
    _check_against_exact(vs, torch, g, qs, k)
    vs.lib().VecSimB200_SetCoarseMode(1)
    single(1, 8)
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
def test_int8_shadow_follows_appends_deletes_reused_ids_and_overwrites():
    """Appends, swap-deletes that move a row with a larger max |x| into another tile (raising its scale), ids re-used by later
    appends: each batch re-quantizes the tiles it must and stays exact.  An in-place overwrite stores a raw row, so the index
    leaves the unit-row copy for the fp16 one and stays exact there."""
    import torch

    from redisearch_b200 import vecsim as vs

    rng = np.random.default_rng(5)
    dim, k, n = 264, 10, 70_000
    rows = ol.synth_rows(ol.F32, 42, 0, n + 2_000, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows[:n], label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, 32, dim)
    _check_against_exact(vs, torch, g, qs, k)
    assert g.add_many(rows[n:n + 1_000], label0=n + 1) == 1_000  # appends into a partial tile and new tiles
    _check_against_exact(vs, torch, g, qs, k)
    spiky = np.zeros(dim, dtype=np.float32)
    spiky[3] = 1.0  # max |x| = 1 after normalisation: every tile this row lands in gets a larger scale
    assert g.add(spiky, n + 5_000) == 1
    for lab in rng.choice(np.arange(1, 1_000), size=40, replace=False):  # swap-deletes: the last rows move into the holes
        assert g.delete(int(lab)) == 1
    _check_against_exact(vs, torch, g, qs, k)
    assert g.add_many(rows[n + 1_000:n + 1_100], label0=n + 10_000) == 100  # ids vacated by the deletes are re-used
    _check_against_exact(vs, torch, g, np.concatenate([qs, spiky[None, :]]), k)
    assert g.add(rows[n + 1_500] * 3.0, 7) == 0  # in-place overwrite of label 7: raw rows from now on
    _check_against_exact(vs, torch, g, qs, k, bits=16)


def _device_index(vs, torch, chunks, dim):
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    n = sum(int(c.shape[0]) for c in chunks)
    assert vs.lib().VecSimB200_Reserve(g.h, n) == 0
    done = 0
    for c in chunks:
        c = (c / c.norm(dim=1, keepdim=True)).contiguous()
        torch.cuda.synchronize()
        assert vs.lib().VecSimB200_AddVectorsDevice(g.h, c.data_ptr(), c.shape[0], done + 1) == c.shape[0]
        done += c.shape[0]
    return g


@pytest.mark.gpu
def test_tier1_proves_every_query_on_uniform_rows_at_1m():
    import torch

    from redisearch_b200 import vecsim as vs

    dim, n, nq, k = 768, 1_048_576, 256, 10
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    chunks = [torch.rand((262_144, dim), generator=gen, device="cuda") * 2 - 1 for _ in range(n // 262_144)]
    g = _device_index(vs, torch, chunks, dim)
    del chunks
    qs = (torch.rand((nq, dim), generator=gen, device="cuda") * 2 - 1).cpu().numpy()
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags == 1).all(), np.bincount(flags)


@pytest.mark.gpu
def test_clustered_corpus_is_proven_by_tiers_1_and_2():
    """Centres with ~1,000 contiguous near-duplicates each (the bench's clustered leg at a quarter of its size): the first tier's
    lists overflow in the centre's row range and the second tier proves the queries."""
    import torch

    from redisearch_b200 import vecsim as vs

    dim, centres_n, per, sigma, nq, k = 768, 500, 1_000, 0.015, 128, 10
    gen = torch.Generator(device="cuda")
    gen.manual_seed(4242)
    centres = torch.rand((centres_n, dim), generator=gen, device="cuda") * 2 - 1
    centres = centres / centres.norm(dim=1, keepdim=True)
    chunks = []
    for c0 in range(0, centres_n, 100):
        which = torch.arange(c0 * per, (c0 + 100) * per, device="cuda") // per
        chunks.append(centres[which] + sigma * torch.randn((100 * per, dim), generator=gen, device="cuda"))
    g = _device_index(vs, torch, chunks, dim)
    del chunks
    qwhich = torch.randint(0, centres_n, (nq,), generator=gen, device="cuda")
    qs = (centres[qwhich] + sigma * torch.randn((nq, dim), generator=gen, device="cuda")).cpu().numpy()
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags != 0).all(), np.bincount(flags)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the planted construction at the k-th boundary, on the int8 route
# ------------------------------------------------------------------------------------------------------------------------------
_NP = 12           # planted queries per corpus, families (a) and (b) alternating: eps_q varies about threefold inside a CTA
_FILL_TILES = 516  # Gaussian filler tiles after the planted ones: 66,048 rows, the route is taken
_corpora = {}


def _clipped(rng, n, dim):
    """Gaussian unit rows with every component within 3 sigma: they never outgrow a planted tile's spike."""
    return _stored(np.clip(rng.standard_normal((n, dim)), -3.0, 3.0).astype(np.float32))


def _decoy(rng, q, dot):
    """A unit row at exact dot product `dot` with q, along q with its components capped at 0.1 (a decoy in a filler tile leaves
    that tile's scale, and delta_max, where the filler has them) plus a random direction orthogonal to both."""
    q64 = q.astype(np.float64)
    w = np.clip(q64, -0.1, 0.1)
    w /= np.linalg.norm(w)
    e1 = q64 / np.linalg.norm(q64)
    e2 = w - (w @ e1) * e1  # zero for a flat query, whose components are all below the cap
    e2 = e2 / np.linalg.norm(e2) if np.linalg.norm(e2) > 1e-9 else e2
    u = rng.standard_normal(q.shape[0])
    u -= (u @ e1) * e1 + (u @ e2) * e2
    u /= np.linalg.norm(u)
    a = dot / float(q64 @ w)
    return (a * w + math.sqrt(1.0 - a * a) * u).astype(np.float32)


def _planted_corpus(dim, nb=129, n_fill_tiles=_FILL_TILES, seed=None):
    """Rows, planted queries and layout.  Planted query i owns tiles 2i and 2i + 1 (tile-aligned, from tile 0 on): A and the first
    127 B rows in the first, the other B rows in the second, clipped Gaussian rows in the rest, all at the scale of SPIKE.  Gaussian filler
    follows.  A filler tile alone would leave the sample pass's k-th smallest distance for a planted query near 0.9 and its
    fixed bound T = a_k + 2 eps_q above half the corpus, so every filler tile also holds one decoy per planted query, a row
    eps_q / 2 farther than its farthest B row: the sample pass then sees at least k of them at every stride, T stays just above
    the planted rows, the lists of 256 hold what passes, and the decoys never enter the top-k."""
    rng = np.random.default_rng(dim if seed is None else seed)
    qs = np.stack([flat_query(rng, dim) if i % 2 == 0 else spiky_query(rng, dim) for i in range(_NP)])
    planted = []
    for i in range(_NP):
        a, b = planted_rows(qs[i], nb)
        t0 = np.concatenate([a[None], b[:127], _clipped(rng, 127 - min(nb, 127), dim)])
        t1 = np.concatenate([b[127:], _clipped(rng, 128 - max(0, nb - 127), dim)])
        planted.append((t0, t1))
    filler = _stored(rng.standard_normal((n_fill_tiles * 128, dim)).astype(np.float32))
    head = np.concatenate([t for pair in planted for t in pair])
    delta_max, x_max = _corpus_stats(np.concatenate([head, filler[:4096]]))
    for i in range(_NP):
        eps = _query_eps(qs[i], delta_max, x_max)[2]
        far = float((planted[i][0][1:].astype(np.float64) @ qs[i].astype(np.float64)).min())
        if nb > 127:
            far = min(far, float((planted[i][1][: nb - 127].astype(np.float64) @ qs[i].astype(np.float64)).min()))
        rows_i = np.arange(n_fill_tiles) * 128 + 8 * i + np.arange(n_fill_tiles) % 8  # one per tile, across its four chunks
        filler[rows_i] = _stored(np.stack([_decoy(rng, qs[i], far - 0.5 * eps) for _ in range(n_fill_tiles)]))
    return np.ascontiguousarray(np.concatenate([head, filler])), qs


def _planted_index(vs, dim):
    if dim not in _corpora:
        rows, qs = _planted_corpus(dim)
        _corpora.clear()  # one corpus at a time on the device
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        assert g.add_many(rows, label0=1) == rows.shape[0]
        p = ol.RefIndex(ol.F32, dim, ol.COS) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
        p.add_many(rows, 1)
        _corpora[dim] = (g, p, qs, rows.shape[0])
    return _corpora[dim]


def _stored_rows(g, n, dim):
    out = np.empty((n, dim), dtype=np.float32)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, out.ctypes.data) == 0
    return out


def _check_power(stored, qs, k, nb=129):
    """The construction's power on the rows the index stores: per planted query, approx(A) - approx(B_k) (distances) against its
    eps_q, with delta_max and x_max over the whole stored corpus."""
    delta_max, x_max = _corpus_stats(stored)
    for i in range(_NP):
        rows = stored[256 * i: 256 * i + 256]
        s_q, _, eps = _query_eps(qs[i], delta_max, x_max)
        approx = 1.0 - _approx(rows, qs[i], s_q)
        ib = np.r_[1:1 + min(nb, 127), 128:128 + max(0, nb - 127)]
        pw = approx[0] - np.sort(approx[ib])[k - 1]
        assert pw >= (1.9 if i % 2 == 0 else 1.0) * eps, (i, pw / eps)


def _sample_stride(tiles, nq, k, sms):
    """sample_stride (vecsim_index.cpp) for the int8 route: the fixed-bound probe's row ranges with 128 queries per CTA."""
    gx = max(1, min(tiles, sms // ((nq + 127) // 128)))
    f = min(0.25, max(0.01, k / (8.0 * gx)))
    return int(max(1.0, min(math.floor(1.0 / f), math.floor(tiles / (2.0 * k)))))


_SLOTS = {16: list(range(12)), 200: [0, 63, 64, 127, 128, 150, 170, 199, 5, 70, 135, 190],
          256: [0, 63, 64, 127, 128, 191, 192, 255, 10, 100, 140, 230],
          1000: [0, 63, 64, 127, 128, 255, 500, 700, 895, 896, 950, 999]}


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nq,k", [(256, 256, 10), (256, 16, 1), (256, 200, 128), (520, 200, 10), (520, 256, 128), (520, 16, 10),
                                      (768, 16, 10), (768, 256, 128), (768, 1000, 10), (768, 200, 1), (768, 256, 10),
                                      (1024, 256, 10), (1024, 200, 128), (1024, 16, 1)])
def test_worst_case_int8_rounding_at_the_kth_boundary(dim, nq, k):
    """Planted queries (planted_rows, families a and b) in both warpgroups of a CTA, both CTAs of a cluster and a partly live last
    CTA, between Gaussian queries.  A is in the reference's top-k, the int8 pass puts it 1.9 eps_q (a) or 1.0 eps_q (b) behind the
    k-th B row, and tier 1 must prove the exact answer.  Tile 0 is in every sample and tiles 1, 3, ... in none at a stride of two
    or more (restated below): with a bound short of the error, the wrong answer is proven in both cases."""
    import torch

    from redisearch_b200 import vecsim as vs

    g, p, pq, n = _planted_index(vs, dim)
    slots = _SLOTS[nq]
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[slots] = pq
    stride = _sample_stride((n + 127) // 128, nq, k, _sm_count(torch))
    assert stride >= 2
    stored = _stored_rows(g, n, dim)
    _check_power(stored, pq, k)
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[slots] == 1).all(), (stride, flags[slots])
    for j, i in enumerate(slots):
        pi, ps = p.topk(qs[i], k)
        assert 256 * j + 1 in pi.tolist(), (j, "A is not in the reference's top-k")
    vs.lib().VecSimB200_SetCoarseMode(1)
    labels, scores, _ = _device_batch(vs, torch, g, _normalized(qs), k)
    vs.lib().VecSimB200_SetCoarseMode(-1)
    for j, i in enumerate(slots):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist() and scores[i].tobytes() == ps.astype(np.float32).tobytes(), (j, i)


def _sm_count(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_worst_case_int8_rounding_in_crowded_ranges_is_proven_by_tier_2():
    """Planted queries of family (b) at batch positions 5 and 70 (both warpgroups of the first CTA) and 130 and 250 (of the second)
    get 384 more rows in one row range of the main pass (three tiles gx apart), farther than every B row by 2.2 eps_q in exact
    terms and inside the fixed bound: their lists overflow, and the second tier's adaptive lists of 128 must still reach A behind
    its B rows.  Queries 0-4 are family (a), with a third of the eps_q: a second tier that read batch query i's bound for open
    query i would cut A off for every crowded query.  The other planted queries of family (a) stay on tier 1."""
    import torch

    from redisearch_b200 import vecsim as vs

    dim, nq, k, nb = 520, 256, 10, 11
    rows, pq = _planted_corpus(dim, nb=nb, seed=77)
    rng = np.random.default_rng(78)
    n = rows.shape[0]
    tiles = (n + 127) // 128
    gx = min(tiles, _sm_count(torch) // ((nq + 127) // 128))  # row ranges of the int8 main pass
    crowded_planted = [1, 3, 5, 7]  # family (b)
    head = 2 * _NP
    delta_max, x_max = _corpus_stats(rows[: head * 128 + 4096])
    for c, i in enumerate(crowded_planted):
        eps = _query_eps(pq[i], delta_max, x_max)[2]
        far = float((rows[256 * i + 1: 256 * i + 1 + nb].astype(np.float64) @ pq[i].astype(np.float64)).min())
        t = head + 3 + 5 * c  # a filler tile; the same range at t + gx and t + 2 gx
        for tt in (t, t + gx, t + 2 * gx):
            rows[tt * 128:(tt + 1) * 128] = _stored(np.stack([_decoy(rng, pq[i], far - 2.2 * eps) for _ in range(128)]))
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    crowded = [5, 70, 130, 250]
    light = [0, 1, 2, 3, 4, 64, 127, 200]
    light_planted = [0, 2, 4, 6, 8, 10, 9, 11]
    qs[crowded] = pq[crowded_planted]
    qs[light] = pq[light_planted]
    _check_power(_stored_rows(g, n, dim), pq, k, nb=nb)
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[crowded] == 2).all(), flags[crowded]
    assert (flags[light[:6]] == 1).all(), flags[light]  # family (a)
    assert (flags[light[6:]] != 0).all(), flags[light]  # family (b) with 11 B rows: proven, on either tier
    p = ol.RefIndex(ol.F32, dim, ol.COS) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
    p.add_many(rows, 1)
    for i, j in zip(crowded + light, crowded_planted + light_planted):
        pi, _ = p.topk(qs[i], k)
        assert 256 * j + 1 in pi.tolist(), (i, "A is not in the reference's top-k")


@pytest.mark.gpu
def test_int8_bound_follows_the_corpus_through_mutations():
    """delta_max is only as good as it is current.  1: the int8 copy built on filler alone; 2: the planted tiles appended (delta_max
    must rise to theirs); 3: more filler appended, a partial refresh that does not touch the planted tiles and must not lower it;
    4: swap-deletes that move a spiky row into a planted tile and raise its scale; 5: more than 256 dirty rows, a full rebuild.
    After every step the planted queries are exact, and proven on tier 1 once their rows are in."""
    import torch

    from redisearch_b200 import vecsim as vs

    dim, k, nq = 256, 10, 16
    rows, pq = _planted_corpus(dim, seed=91)
    head = 2 * _NP * 128
    planted, filler = rows[:head], rows[head:]
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[: _NP] = pq
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(filler, label0=1) == filler.shape[0]
    _check_against_exact(vs, torch, g, qs, k)  # 1
    lab = filler.shape[0] + 1
    assert g.add_many(planted, label0=lab) == head  # 2: tile-aligned, A of planted query i is label lab + 256 i
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[: _NP] == 1).all(), flags
    more = _stored(np.random.default_rng(92).standard_normal((2 * 128, dim)).astype(np.float32))
    assert g.add_many(more, label0=lab + head) == more.shape[0]  # 3
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[: _NP] == 1).all(), flags
    spiky = np.zeros(dim, dtype=np.float32)
    spiky[7] = 0.9
    spiky[8] = math.sqrt(1 - 0.81)
    assert g.add(spiky, lab + head + 10_000) == 1  # the last row ...
    assert g.delete(lab + 128 + 100) == 1  # ... moves into the second tile of planted query 0, a clipped Gaussian row's place,
    # and the two B rows there lose their midpoints
    flags = _check_against_exact(vs, torch, g, qs, k)  # 4
    assert (flags[: _NP] == 1).all(), flags
    for j in range(300):  # 5: swap-deletes of filler rows, each dirtying the hole it leaves
        assert g.delete(1 + 200 * j) == 1
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[: _NP] == 1).all(), flags
