"""The batched fp32 KNN route (fp16 GEMM -> rows under a bound -> exact rescoring -> proof, DESIGN.md §4) against inputs
built to break it: rows whose 16-bit operand form rounds their dot product with the query the wrong way by as much as the
format allows, values at the edges of the fp16 range, queries outside it, and candidate counts at the list capacity.

Random rows use under a tenth of the error bound eps, so a suite of random data passes with eps divided by eight.  The
builders below place every component of a row just short of a rounding point of the operand format, on the side that
moves the dot product against (or with) the query; a CPU test checks that they keep that power.

Every GPU case compares ids and score bits with the reference (its compiled code when oracle/_ref is built, else the C
restatement at the AVX-512 tier) and checks that the batch ran the tensor-core route (LastBatchPath == 1).
"""
import ctypes as C
import math

import numpy as np
import pytest

import oracle_lib as ol

EPS_F16, EPS_TF32 = 1.2e-3, 2.5e-3  # kCoarseEpsF16 / kCoarseEpsTF32 (csrc/coarse_tc.h)


# ------------------------------------------------------------------------------------------------------------------
# numpy emulation of the coarse GEMM and of its error bound
# ------------------------------------------------------------------------------------------------------------------
def _f16(x):
    """fp32 -> fp16, round to nearest even (to_f16_kernel), as float64."""
    return np.asarray(x, dtype=np.float32).astype(np.float16).astype(np.float64)


def _tf32(x):
    """fp32 -> the 10-bit mantissa the TF32 MMA reads: the low 13 bits are dropped (truncation)."""
    u = np.ascontiguousarray(np.asarray(x, dtype=np.float32)).view(np.uint32) & np.uint32(0xFFFFE000)
    return u.view(np.float32).astype(np.float64)


def approx_dist(rows, q, metric, kind="f16"):
    """Approximate distances of the coarse pass: 16-bit operands, exact (float64) accumulation; squared L2 takes the
    exact squared norms, as the kernel's epilogue does."""
    cv = _f16 if kind == "f16" else _tf32
    dot = cv(rows) @ cv(q)
    if metric == ol.L2:
        r64, q64 = np.asarray(rows, np.float64), np.asarray(q, np.float64)
        return (r64 * r64).sum(axis=-1) + q64 @ q64 - 2.0 * dot
    return 1.0 - dot


def exact_dist(rows, q, metric):
    r64, q64 = np.asarray(rows, np.float64), np.asarray(q, np.float64)
    if metric == ol.L2:
        d = r64 - q64
        return (d * d).sum(axis=-1)
    return 1.0 - r64 @ q64


def query_eps(eps, max_norm, q_norm, dim, l2, subnormal_term=True):
    """query_eps of csrc/coarse_tc.cu (norm-scaled bound of raw inner product / L2)."""
    e = eps * max_norm * q_norm + (5.97e-8 * math.sqrt(dim) * (max_norm + q_norm) if subnormal_term else 0.0)
    if l2:
        e = 2.0 * e + (dim + 4) * 1.2e-7 * (max_norm * max_norm + q_norm * q_norm)
    return e * 1.0001


def power(stored_a, stored_b, q, metric, k, kind="f16"):
    """approx(A) - (k-th smallest approx over the B rows): how far the worst-case rounding pushes the true top-k row A
    behind k rows it beats in exact arithmetic."""
    pa = approx_dist(stored_a, q, metric, kind)
    pb = np.sort(approx_dist(stored_b, q, metric, kind))
    return float(pa - pb[k - 1])


# ------------------------------------------------------------------------------------------------------------------
# builders
# ------------------------------------------------------------------------------------------------------------------
def adversarial_unit_rows(q, nb, kind="f16"):
    """Row A and nb rows B for the unit query q: A's exact dot product with q is above every B's (by under 2e-4), but
    the operand form (kind "f16": round to nearest; "tf32": truncation) moves A's dot down and the B rows' up by nearly
    the most the format allows.

    Every component but one sits at the bottom of a binade of the format, where half an ulp is the largest fraction
    of the value (2^-11 of it), signed like q, and just short of a rounding point: below it for A, above it for B.
    The component with the smallest |q_i| absorbs the norm, so the rows are unit vectors to fp32 precision and the
    cosine index stores them unchanged but for a unit or two in the last place.  Returns (A [dim], B [nb, dim]) fp32."""
    q = np.asarray(q, np.float64)
    dim = q.shape[0]
    order = np.argsort(-np.abs(q), kind="stable")
    slack = order[-1]
    e0 = math.floor(math.log2(1.0 / math.sqrt(dim)))
    lo, hi = 2.0 ** e0, 2.0 ** (e0 + 1)
    n_hi = int((0.97 - (dim - 1) * lo * lo) / (hi * hi - lo * lo))
    base = np.full(dim, lo)
    base[order[:n_hi]] = hi                # the largest |q_i| get the larger magnitude
    ulp = base * 2.0 ** -10                # both formats keep 10 mantissa bits
    half = 0.5 if kind == "f16" else 1.0   # rounding point: the midpoint (nearest) or the next value (truncation)
    tiny = base * 2.0 ** -20               # 8 fp32 ulps: the cosine index's renormalisation moves a component by <= 2
    top = order[:8]
    sign = np.where(q < 0, -1.0, 1.0)

    def row(jset, against):
        j = np.zeros(dim)
        j[top[[b for b in range(8) if jset >> b & 1]]] = 1.0  # one ulp more on a subset of the top components
        mag = base + ulp * (j + half) + (-tiny if against else tiny)
        mag[slack] = 0.0
        mag[slack] = math.sqrt(1.0 - float((mag * mag).sum()))
        return (sign * mag).astype(np.float32)

    assert nb < 255
    a = row(255, True)                          # all eight: A has the largest exact dot product
    b = np.stack([row(m, False) for m in range(nb)])
    return a, b


def adversarial_subnormal_rows(q, nb):
    """Row A and nb rows B for a query q whose components lie in the fp16 subnormal range: components near 2e-6 (the
    fp16 grid there is 2^-24), signed like q, just short of a grid midpoint (A below, B above).  A is the nearest in
    exact arithmetic (one grid step more on the top components); the fp16 GEMM moves A's dot product down and the B
    rows' up by 2^-25 per component — relative to the tiny norms far more than eps * |a| * |q|, which is why query_eps
    carries a 2^-24 sqrt(D) term.  Returns (A, B) fp32."""
    q = np.asarray(q, np.float64)
    dim = q.shape[0]
    order = np.argsort(-np.abs(q), kind="stable")
    top = order[:8]
    g = 2.0 ** -24
    sign = np.where(q < 0, -1.0, 1.0)

    def row(jset, against):
        j = np.full(dim, 33.0)
        j[top[[b for b in range(8) if jset >> b & 1]]] += 1.0
        mag = g * (j + 0.5) + (-g if against else g) * 2.0 ** -10
        return (sign * mag).astype(np.float32)

    return row(255, True), np.stack([row(m, False) for m in range(nb)])


def subnormal_query(rng, dim):
    return (np.where(rng.random(dim) < 0.5, -1.0, 1.0) * rng.uniform(1e-5, 5e-5, dim)).astype(np.float32)


def _unit_query(rng, dim):
    q = rng.standard_normal(dim)
    return (q / np.linalg.norm(q)).astype(np.float32)


def _normalized(x):
    """The reference's normalisation (the C restatement of it) of fp32 rows, as a cosine index stores them."""
    x = np.array(x, dtype=np.float32, copy=True)
    for r in np.atleast_2d(x):
        ol.port().orc_normalize(ol._p(r), r.shape[0], ol.F32)
    return x


# ------------------------------------------------------------------------------------------------------------------
# CPU: the builders keep their power
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [128, 768])
def test_adversarial_builders_have_power(dim):
    rng = np.random.default_rng(dim)
    k = 10
    for _ in range(4):
        q = _normalized(_unit_query(rng, dim))
        for kind, eps, need in (("f16", EPS_F16, EPS_F16 / 2), ("tf32", EPS_TF32, EPS_TF32 / 4)):
            a, b = adversarial_unit_rows(q, k + 2, kind)
            sa, sb = _normalized(a), _normalized(b)  # what a cosine index stores
            ea, eb = exact_dist(sa, q, ol.COS), exact_dist(sb, q, ol.COS)
            assert ea < eb.min(), "A must be the best of the planted rows in exact arithmetic"
            assert eb.max() - ea < 2e-4  # B is only slightly worse
            # the worst-case rounding puts A behind all k rows B by at least `need` (TF32: truncation of a unit vector
            # moves a dot product by at most 2^-10 of it, so eps_tf32 / 2 is out of reach; eps_tf32 / 4 is not)
            p = power(sa, sb, q, ol.COS, k, kind)
            assert p >= need, (kind, p, need)
            # ... and never by more than the bound the proof uses
            assert abs(approx_dist(sa, q, ol.COS, kind) - ea) <= eps and np.abs(approx_dist(sb, q, ol.COS, kind) - eb).max() <= eps
        # raw inner product / L2: the same rows scaled by a power of two round the same way; the power scales with the norms
        for metric in (ol.IP, ol.L2):
            s = 8.0
            a, b = adversarial_unit_rows(q, k + 2)
            qs = (s * q.astype(np.float64)).astype(np.float32)
            ra, rb = (s * a.astype(np.float64)).astype(np.float32), (s * b.astype(np.float64)).astype(np.float32)
            mx = float(np.sqrt(max((ra.astype(np.float64) ** 2).sum(), (rb.astype(np.float64) ** 2).sum(1).max())))
            e = query_eps(EPS_F16, mx, float(np.linalg.norm(qs.astype(np.float64))), dim, metric == ol.L2)
            assert exact_dist(ra, qs, metric) < exact_dist(rb, qs, metric).min()
            assert power(ra, rb, qs, metric, k) >= e / 2, (metric, power(ra, rb, qs, metric, k), e)


@pytest.mark.parametrize("dim", [128, 768])
def test_subnormal_builder_exceeds_the_bound_without_its_subnormal_term(dim):
    rng = np.random.default_rng(7 + dim)
    for _ in range(4):
        q = subnormal_query(rng, dim)
        a, b = adversarial_subnormal_rows(q, 12)
        assert (np.abs(a) >= 1e-6).all() and (np.abs(a) < 6e-5).all() and (np.abs(q) < 6e-5).all()
        assert exact_dist(a, q, ol.L2) < exact_dist(b, q, ol.L2).min()
        mx = float(np.sqrt(max((a.astype(np.float64) ** 2).sum(), (b.astype(np.float64) ** 2).sum(1).max())))
        qn = float(np.linalg.norm(q.astype(np.float64)))
        full = query_eps(EPS_F16, mx, qn, dim, True)
        bare = query_eps(EPS_F16, mx, qn, dim, True, subnormal_term=False)
        err = abs(float(approx_dist(a, q, ol.L2)) - float(exact_dist(a, q, ol.L2)))
        assert err > bare, (err, bare)   # without the 2^-24 sqrt(D) term the bound would not hold ...
        assert err <= full, (err, full)  # ... with it, it does
        assert power(a, b, q, ol.L2, 10) > 2 * bare  # so the cut a_k + 2 eps would drop A


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _checker(metric, dim):
    if ol.ref_vecsim() is not None:
        return ol.RefIndex(ol.F32, dim, metric)
    return ol.PortIndex(ol.F32, dim, metric, tier=ol.TIER_AVX512)


def _device_batch(vs, index, qs, k):
    import torch

    nq = qs.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qs, dtype=np.float32)).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert vs.lib().VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)
    return out_l.cpu().numpy(), out_s.cpu().numpy(), (flags if frc == 0 else None)


def _read_rows(index, rows, dim):
    out = np.empty((len(rows), dim), dtype=np.float32)
    for i, r in enumerate(rows):
        assert index.L.VecSimB200_ReadRows(index.h, int(r), 1, out[i].ctypes.data) == 0
    return out


def _assert_exact(labels, scores, p, qs_raw, k, flags=None, what=""):
    for i in range(qs_raw.shape[0]):
        pi, ps = p.topk(qs_raw[i], k)
        assert labels[i].tolist() == pi.tolist(), (what, i, None if flags is None else int(flags[i]), labels[i][:12], pi[:12])
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes(), (what, i)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _metric_code(vs, metric):
    return {ol.L2: vs.VecSimMetric_L2, ol.IP: vs.VecSimMetric_IP, ol.COS: vs.VecSimMetric_Cosine}[metric]


# ------------------------------------------------------------------------------------------------------------------
# GPU: worst-case rounding at the k-th boundary
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [10, 100])
@pytest.mark.parametrize("dim", [128, 768])
@pytest.mark.parametrize("case", ["cos_f16", "cos_tf32", "ip", "l2"])
def test_worst_case_rounding_at_the_kth_boundary(case, dim, k):
    """Per query: row A is in the true top-k but its operand form rounds it behind k + 1 rows B it beats in exact
    arithmetic (by at least eps / 2 in the emulated GEMM; TF32: eps / 4).  The refine cut a_k + 2 eps must still reach A,
    and the proof must hold; with a smaller eps A is dropped and the proof passes on a wrong answer.  The batch must read
    the copy the emulation models (fp16: 16 bits; TF32 reads the fp32 rows: 0).  Unit cosine rows wider than 128 dimensions
    take the int8 copy on a single-value index (test_coarse_int8_shadow.py holds that route to its own worst case), so
    cos_f16 at 768 runs on a multi-value index with one row per label: it keeps the fp16 copy and answers what the
    single-value index answers."""
    from redisearch_b200 import vecsim as vs

    metric = {"cos_f16": ol.COS, "cos_tf32": ol.COS, "ip": ol.IP, "l2": ol.L2}[case]
    kind = "tf32" if case == "cos_tf32" else "f16"
    vs.lib().VecSimB200_SetCoarseMode(2 if kind == "tf32" else 1)
    n, nq = 70_000, 16
    rng = np.random.default_rng(1000 * dim + k)
    rows = ol.synth_rows(ol.F32, 61, 0, n, dim)
    raw_q = np.stack([_unit_query(rng, dim) for _ in range(nq)])
    qn = _normalized(raw_q) if metric == ol.COS else raw_q
    # raw inner product / L2: the planted rows carry the corpus's largest norm (a power of two keeps their rounding),
    # and the queries the same norm, so that the dot term dominates the L2 bound
    scale = 1.0 if metric == ol.COS else 2.0 ** math.ceil(math.log2(float(np.sqrt((rows.astype(np.float64) ** 2).sum(1).max()))))
    qdev = (qn.astype(np.float64) * scale).astype(np.float32) if metric != ol.COS else qn
    nb = k + 1
    pos = rng.permutation(n)[: nq * (nb + 1)].reshape(nq, nb + 1)  # spread over the row ranges: no list overflows
    for i in range(nq):
        a, b = adversarial_unit_rows(qn[i], nb, kind)
        rows[pos[i, 0]] = (a.astype(np.float64) * scale).astype(np.float32)
        rows[pos[i, 1:]] = (b.astype(np.float64) * scale).astype(np.float32)
    multi = case == "cos_f16" and dim > 128
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric), multi=multi)
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs_raw = raw_q if metric == ol.COS else qdev
    labels, scores, flags = _device_batch(vs, g, qdev, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    assert vs.lib().VecSimB200_LastCoarseShadowBits(g.h) == (0 if kind == "tf32" else 16)
    assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags, minlength=4).tolist()
    _assert_exact(labels, scores, p, qs_raw, k, flags, case)
    # the construction has power on the rows the index actually stores (cosine: after its normalisation)
    if metric == ol.COS:
        max_norm = None
    else:
        max_norm = float(np.sqrt(np.max((rows.astype(np.float64) ** 2).sum(1))))
    eps = EPS_TF32 if kind == "tf32" else EPS_F16
    for i in range(nq):
        pi, _ = p.topk(qs_raw[i], k)
        assert pos[i, 0] + 1 in pi.tolist(), (i, "A is not in the reference's top-k")
        st = _read_rows(g, pos[i], dim)
        q64 = qdev[i]
        if max_norm is None:
            e = eps
        else:
            e = query_eps(eps, max_norm, float(np.linalg.norm(q64.astype(np.float64))), dim, metric == ol.L2)
        need = e / 4 if kind == "tf32" else e / 2
        pw = power(st[0], st[1:], q64, metric, k, kind)
        assert pw >= need, (i, pw, need)
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: dynamic range
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.L2])
def test_sift_like_rows_with_large_norms_and_offset(metric):
    """Non-negative integer components 0..255 (SIFT-like): norms near 1,500 and a large common offset."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 128, 32, 10
    rows = np.rint((ol.synth_rows(ol.F32, 71, 0, n, dim) + 1.0) * 127.5).astype(np.float32)
    qs = np.rint((ol.synth_rows(ol.F32, 72, 0, nq, dim) + 1.0) * 127.5).astype(np.float32)
    qs[: nq // 2] = rows[1000: 1000 + nq // 2] + 1.0  # queries next to stored rows
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    labels, scores, flags = _device_batch(vs, g, qs, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    _assert_exact(labels, scores, p, qs, k, flags, "sift")
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.L2])
def test_subnormal_rows_and_queries_rounded_adversarially(metric):
    """Every component in the fp16 subnormal range (1e-6 .. 6e-5), the planted rows rounded against / with the query:
    the fp16 error of a row is far above eps |a| |q|, only the 2^-24 sqrt(D) term of query_eps covers it.  (Inner product
    distances 1 - dot are all 1.0f here: a corpus of ties, which the proof must not pass.)"""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 128, 16, 10
    rng = np.random.default_rng(81)
    x = ol.synth_rows(ol.F32, 82, 0, n, dim)
    rows = (np.sign(x) * (1e-6 + 1e-6 * np.abs(x))).astype(np.float32)
    qs = np.stack([subnormal_query(rng, dim) for _ in range(nq)])
    nb = k + 2
    pos = rng.permutation(n)[: nq * (nb + 1)].reshape(nq, nb + 1)
    for i in range(nq):
        a, b = adversarial_subnormal_rows(qs[i], nb)
        rows[pos[i, 0]] = a
        rows[pos[i, 1:]] = b
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    labels, scores, flags = _device_batch(vs, g, qs, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    _assert_exact(labels, scores, p, qs, k, flags, "subnormal")
    if metric == ol.L2:
        assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags, minlength=3).tolist()
        max_norm = float(np.sqrt(np.max((rows.astype(np.float64) ** 2).sum(1))))
        for i in range(nq):
            assert labels[i, 0] == pos[i, 0] + 1
            bare = query_eps(EPS_F16, max_norm, float(np.linalg.norm(qs[i].astype(np.float64))), dim, True, subnormal_term=False)
            assert power(rows[pos[i, 0]], rows[pos[i, 1:]], qs[i], ol.L2, k) > 2 * bare
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.L2])
def test_fp16_range_limit_of_the_rows(metric):
    """A component of exactly 60000 keeps the index on the route; the next float above it sends the index to the exact
    scan.  Either way the answer is the reference's."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 64, 16, 10
    qs = ol.synth_rows(ol.F32, 92, 0, nq, dim)
    for value, path in ((np.float32(60000.0), 1), (np.nextafter(np.float32(60000.0), np.float32(np.inf)), 0)):
        rows = ol.synth_rows(ol.F32, 91, 0, n, dim)
        rows[4321, 7] = value
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
        p = _checker(metric, dim)
        assert g.add_many(rows, label0=1) == n
        p.add_many(rows, 1)
        labels, scores, flags = _device_batch(vs, g, qs, k)
        assert vs.lib().VecSimB200_LastBatchPath(g.h) == path, float(value)
        assert (flags is not None) == (path == 1)
        _assert_exact(labels, scores, p, qs, k, flags, float(value))
        g.close()
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: queries outside the fp16 range
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [ol.IP, ol.L2])
def test_queries_outside_the_fp16_range_are_never_proven(metric):
    """A query component of 65520 or more is +-inf in fp16, so every approximate distance of that query is +-inf or NaN
    and no error bound holds.  The trap: component 0 is -2^-20 on every row except 20 bait rows in row tile 1, where it
    is +2^-20.  For q_0 >= 65520 the bait rows get approximate distance -inf and every other row +inf.  The sample pass
    visits every stride-th tile (stride >= 2 at this size, so never tile 1) and sees only +inf, the bound is +inf, the
    main pass keeps the bait rows alone, and a proof that trusted those numbers would return them.  In exact arithmetic
    the bait rows are not the answer.  Such queries must be answered by the exact scan (flag 0), while the ordinary
    queries of the same batch and the one at 65504 (finite in fp16) stay proven on the tensor-core tiers."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 64, 16, 10
    rows = ol.synth_rows(ol.F32, 101, 0, n, dim)
    tiny = np.float32(2.0 ** -20)  # an fp16 subnormal: inf * it is inf, not NaN
    rows[:, 0] = -tiny
    bait = np.arange(128, 148)
    rows[bait, 0] = tiny
    # the query at -65504 has its answer in 10 rows with a large negative component 0 (a clear margin for the proof)
    win = np.arange(30_000, 30_000 + 4 * k, 4)
    rows[win, 0] = -(4.0 + 0.25 * np.arange(k)).astype(np.float32)
    qs = ol.synth_rows(ol.F32, 102, 0, nq, dim)
    big = {0: -65504.0, 1: 65520.0, 2: 1e5, 3: 1e30}
    for i, v in big.items():
        qs[i, 0] = np.float32(v)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    labels, scores, flags = _device_batch(vs, g, qs, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    report = []
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        if labels[i].tolist() != pi.tolist() or scores[i].tobytes() != ps.astype(np.float32).tobytes():
            report.append(f"query {i} (q_0 = {float(qs[i, 0]):g}): flag {int(flags[i])}, ids {labels[i].tolist()}, reference {pi.tolist()}")
    assert not report, "\n".join(report)
    assert sorted(labels[0].tolist()) == sorted((win + 1).tolist())
    assert (flags[1:4] == 0).all(), flags.tolist()
    assert flags[0] != 0 and (flags[4:] != 0).all(), flags.tolist()
    # single queries ride the shadow the batch built, under the same rule
    for i in range(nq):
        gi, gs, code = g.topk(qs[i], k)
        pi, ps = p.topk(qs[i], k)
        assert code == 0 and gi.tolist() == pi.tolist() and gs.astype(np.float32).tobytes() == ps.astype(np.float32).tobytes(), i
        assert vs.lib().VecSimB200_LastBatchPath(g.h) == (0 if i in (1, 2, 3) else 1), i
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the fragment epilogue of the fixed-bound main pass
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nq", [64, 255, 257, 320])
@pytest.mark.parametrize("metric", [ol.COS, ol.L2])
def test_every_fragment_position_reaches_the_lists(metric, nq):
    """The main pass tests the bound on the m64n128 accumulator fragment.  Query i's true top-128 sit at row offset m of
    tile (i + m) mod tiles for m = 0..127, so together the queries cover every (query slot, row offset) pair of the
    fragment; nq covers partial query groups and cluster sizes 1, 2 and 4.  n is odd: L2 loads the squared norms of row
    pairs as one float2, and query 0's three nearest rows are n - 1, n - 2 and the first row of the partial last tile."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, k = 70_001, 64, 128
    tiles = (n + 127) // 128
    rng = np.random.default_rng(nq)
    rows = ol.synth_rows(ol.F32, 111, 0, n, dim)
    qs = ol.synth_rows(ol.F32, 112, 0, nq, dim)
    if metric == ol.COS:
        qn = _normalized(qs)
    m = np.arange(128)
    for i in range(nq):
        at = ((i + m) % (tiles - 1)) * 128 + m  # never the partial last tile
        u = rng.standard_normal((128, dim))
        if metric == ol.COS:
            u -= (u @ qn[i].astype(np.float64))[:, None] * qn[i].astype(np.float64)[None, :]
            u /= np.linalg.norm(u, axis=1, keepdims=True)
            c = 0.95 - 0.001 * rng.permutation(128)  # distinct, spread over the offsets
            rows[at] = (c[:, None] * qn[i].astype(np.float64)[None, :] + np.sqrt(1 - c * c)[:, None] * u).astype(np.float32)
        else:
            r = 0.05 + 0.002 * rng.permutation(128)
            rows[at] = (qs[i].astype(np.float64)[None, :] + r[:, None] * u / np.linalg.norm(u, axis=1, keepdims=True)).astype(np.float32)
    last = (tiles - 1) * 128
    for j, r in enumerate((n - 1, n - 2, last)):
        rows[r] = (qs[0].astype(np.float64) + 1e-3 * (j + 1) * rng.standard_normal(dim) / math.sqrt(dim)).astype(np.float32)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, _metric_code(vs, metric))
    p = _checker(metric, dim)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    labels, scores, flags = _device_batch(vs, g, qn if metric == ol.COS else qs, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags, minlength=3).tolist()
    _assert_exact(labels, scores, p, qs, k, flags, f"nq {nq}")
    if metric == ol.L2:
        assert set(labels[0, :3].tolist()) == {n, n - 1, last + 1}
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: candidate counts across the list capacity
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sweep_across_the_list_capacity():
    """Per query, csz near-duplicates in one row tile the sample pass visits plus the query's own vector in a later
    tile of the same row range: csz + 1 rows of that range fall below the bound.  Up to 96 (the list capacity) the first
    tier proves the answer; from 97 on the list overflows and the second tier must answer — a list that silently
    dropped its last append would lose the nearest row, which arrives last."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 128, 16, 10
    tiles = (n + 127) // 128
    stride = max(1, min(100, tiles // (2 * k)))  # batch_scan: the sample fraction is clamped to 0.01 at this size
    gx = min(tiles, torch.cuda.get_device_properties(0).multi_processor_count)  # row ranges of the main pass (nq <= 64)
    assert (nq - 1) * stride + gx < tiles
    n_sampled = (tiles + stride - 1) // stride  # tiles 0, stride, 2 stride, ...
    tiers = set()
    for csz in range(80, 113, 4):
        rng = np.random.default_rng(csz)
        rows = ol.synth_rows(ol.F32, 121, 0, n, dim)
        qs = np.empty((nq, dim), dtype=np.float32)
        for i in range(nq):
            t = i * stride  # a sampled tile
            center = rng.uniform(-1, 1, dim)
            rows[t * 128: t * 128 + csz] = (center[None, :] + 1e-3 * rng.standard_normal((csz, dim))).astype(np.float32)
            qs[i] = (center + 1e-3 * rng.standard_normal(dim)).astype(np.float32)
            rows[(t + gx) * 128 + 5] = qs[i]  # same row range, a later tile: appended last
            # k more near-duplicates in k other sampled tiles: the sample pass keeps one minimum per 32-row chunk, so these
            # put its k-th smallest, and the bound, within 2 eps of the cluster — no unrelated row of the range is below it
            for j in range(1, k + 1):
                rows[((i + j) % n_sampled) * stride * 128 + 112 + i] = (center + 1e-3 * rng.standard_normal(dim)).astype(np.float32)
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        p = _checker(ol.COS, dim)
        assert g.add_many(rows, label0=1) == n
        p.add_many(rows, 1)
        labels, scores, flags = _device_batch(vs, g, _normalized(qs), k)
        assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
        _assert_exact(labels, scores, p, qs, k, flags, f"csz {csz}")
        want = 1 if csz + 1 <= 96 else 2
        assert (flags == want).sum() >= nq * 0.9, (csz, np.bincount(flags, minlength=3).tolist())
        tiers.update(int(f) for f in flags)
        g.close()
    assert {1, 2} <= tiers
    vs.lib().VecSimB200_SetCoarseMode(-1)
