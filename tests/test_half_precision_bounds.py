"""fp16 / bf16 KNN against float64 distances of the stored values, with derived error bounds, on every search path.

The BASELINE bar for 16-bit corpora (scores within 1e-2, ids equal modulo candidates within 1e-2 of the k-th) cannot see a
kernel that accumulates in fp16, a selection that returns the 11th row instead of the 10th, a score attached to the wrong
label, or a route that drops rows tied with its bound.  This file holds every 16-bit path to a bar derived from the arithmetic:

  * the stored rows are read back from HBM (VecSimB200_ReadRows) and the stored query is the library's own normalised blob;
    both are decoded exactly to float64 and give e = 1 - sum x_i y_i (IP / cosine) or sum (x_i - y_i)^2 (L2), exactly enough;
  * every returned score must lie within B of e, B being the worst-case rounding error of the arithmetic the path performs
    (bound_cuda_core, bound_tensor_core); the largest |score - e| / B each test sees is printed;
  * the ids must be consistent with e: every label clearly inside the k-th distance is returned, nothing clearly outside is;
  * the CUDA-core paths (DistTile16) sum in an order that does not depend on the tile shape, so every one of them must give
    the same bits for the same (row, query), and their answers must be exactly the (score, label) selection over those bits.

Multi-value indexes fold a label's rows with the reference's float rule (brute_force_multi.h:234-238), NaN included.
The tests without the gpu marker hold the checker itself to simulated wrong answers: it must reject each of them.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as ol
from oracle_lib import BF16, COS, F16, IP, L2
from test_vecsim_parity import DIM_SWEEP

U = 2.0 ** -24  # unit roundoff of fp32
VT = {F16: 3, BF16: 2}
MT = {L2: 0, IP: 1, COS: 2}
TNAME = {F16: "fp16", BF16: "bf16"}
MNAME = {L2: "L2", IP: "IP", COS: "COS"}
SIZE_MAX = np.uint64(0xFFFFFFFFFFFFFFFF)


# ------------------------------------------------------------------------------------------------------------------
# the reference: exact distances of the stored values, and the bounds
# ------------------------------------------------------------------------------------------------------------------
def decode16(bits, vtype):
    """16-bit blobs -> float64, exactly (every fp16 / bf16 value is a float64)."""
    bits = np.ascontiguousarray(bits, dtype=np.uint16)
    if vtype == F16:
        return bits.view(np.float16).astype(np.float64)
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def to16(x32, vtype):
    """float32 values -> fp16 / bf16 bits, round to nearest even (numpy's half; bfloat16.h:22-29 for bf16, as ol.to_type)."""
    x32 = np.ascontiguousarray(x32, dtype=np.float32)
    if vtype == F16:
        return x32.astype(np.float16).view(np.uint16)
    b = x32.view(np.uint32)
    return ((b + ((b >> 16) & 1) + np.uint32(0x7FFF)) >> 16).astype(np.uint16)


def exact_distances(X, y, metric):
    """(e, mag) of every row of X (float64) against y: e the distance in float64, mag = sum |x_i y_i| (IP / cosine) or
    sum (x_i - y_i)^2 (L2), the magnitude the rounding errors scale with."""
    if metric == L2:
        d = X - y
        e = np.einsum("ij,ij->i", d, d)
        return e, e
    p = X * y
    return 1.0 - p.sum(axis=1), np.abs(p).sum(axis=1)


def gamma(n):
    return n * U / (1.0 - n * U)


def chain_length(dim):
    """fmaf steps of one lane in DistTile16: 8 per 16-byte vector it owns (lane l owns vectors l, l + 32, ...), plus one
    for the scalar tail (dim mod 8 elements, one per lane)."""
    return 8 * math.ceil((dim // 8) / 32) + math.ceil((dim % 8) / 32)


def bound_cuda_core(e, mag, dim):
    """|score - e| for DistTile16 (scan_topk, scan_scores, gather, gather_min).

    Each lane runs one fmaf chain of length m = chain_length(dim) over exact operands (fp16 / bf16 -> fp32 is exact), and
    the 32 lane sums meet in 5 butterfly adds, so every term passes through at most m + 5 roundings; for L2 the difference
    x - y and its square add two more (the square is folded into the fma, the difference rounds once, and (1 + d)^2 is
    within two roundings).  The standard recursive-summation bound (Higham, Accuracy and Stability of Numerical
    Algorithms, 3.1 and 4.2) gives |acc - sum| <= gamma_{m+7} * sum |terms| = gamma_{m+7} * mag.  IP / cosine subtract the
    sum from 1 once more (u |e|).  fp32 underflow of a product or a partial sum costs at most 2^-150 per step, hence
    dim * 2^-149.  At dim 768 this is about 2e-6 * mag."""
    return gamma(chain_length(dim) + 7) * mag + U * np.abs(e) + dim * 2.0 ** -149


def bound_tensor_core(e, mag, dim):
    """|score - e| for the direct 16-bit wgmma route.  Products of 16-bit operands are exact in the fp32 accumulator; the
    bound assumes each accumulation step loses at most 2^-23 relative to the running magnitude (aligned and truncated), so
    dim steps lose dim * 2^-23 * mag, doubled for the final alignment of the partial sums, plus u |e| for 1 - dot.  This is
    an assumption about Hopper's wgmma adder, measured (not derived) by the tests that print err / B for this route."""
    return dim * 2.0 ** -22 * mag + U * np.abs(e)


def check_answer(labels, scores, e_of, b_of, k, tie_order=True):
    """One query's (labels, scores) against the exact distances.  e_of / b_of: float64 arrays indexed by label, NaN where
    there is no label.  A label whose e is not finite (fp32 overflow) must carry that very value.  Returns max err / B."""
    labels = np.asarray(labels, dtype=np.int64)
    scores = np.asarray(scores, dtype=np.float64)
    valid = ~np.isnan(e_of)
    n_labels = int(valid.sum())
    assert len(labels) == min(k, n_labels), (len(labels), k, n_labels)  # 5. the count
    if not len(labels):
        return 0.0
    assert len(set(labels.tolist())) == len(labels), "a label is returned twice"
    assert valid[labels].all(), "a returned label is not in the index"
    e, b = e_of[labels], b_of[labels]
    fin = np.isfinite(e)
    assert (scores[~fin] == e[~fin]).all(), (labels[~fin], scores[~fin], e[~fin])
    err = np.abs(scores[fin] - e[fin])
    bad = err > b[fin]
    assert not bad.any(), ("score outside the bound", labels[fin][bad][:5], scores[fin][bad][:5], e[fin][bad][:5], b[fin][bad][:5])  # 1.
    s32 = scores.astype(np.float32)
    assert (s32[1:] >= s32[:-1]).all(), "scores are not non-decreasing"  # 2.
    if tie_order:
        tied = s32[1:] == s32[:-1]
        assert (labels[1:][tied] > labels[:-1][tied]).all(), "bit-equal scores out of label order"
    kk = len(labels)
    ev = e_of[valid]
    ek = np.partition(ev, kk - 1)[kk - 1]
    if np.isfinite(ek):
        top = valid & (e_of <= ek)
        bmax = max(float(np.max(b_of[top])), float(np.max(b)))
        must = np.flatnonzero(valid & (e_of < ek - 2 * bmax))
        missing = set(must.tolist()) - set(labels.tolist())
        assert not missing, ("clearly inside the k-th distance, not returned", sorted(missing)[:5], ek, bmax)  # 3.
        assert (e <= ek + 2 * bmax).all(), ("clearly outside the k-th distance, returned", labels[e > ek + 2 * bmax][:5])  # 4.
    return float((err / b[fin]).max()) if fin.any() else 0.0


def per_label(e_rows, b_rows, row_labels, size):
    """Multi-value index: e of a label = min over its rows, its bound the largest of its rows' bounds."""
    e_of = np.full(size, np.inf)
    b_of = np.zeros(size)
    np.minimum.at(e_of, row_labels, e_rows)
    np.maximum.at(b_of, row_labels, b_rows)
    seen = np.zeros(size, dtype=bool)
    seen[row_labels] = True
    e_of[~seen] = np.nan
    return e_of, b_of


def reference_fold(ds):
    """getDistanceFrom_Unsafe of a multi-value index (brute_force_multi.h:234-238), in float."""
    dist = np.float32(np.inf)
    for d in ds:
        d = np.float32(d)
        dist = dist if dist < d else d
    return dist


# ------------------------------------------------------------------------------------------------------------------
# CPU: the checker rejects wrong answers and accepts right ones (numpy-simulated kernels)
# ------------------------------------------------------------------------------------------------------------------
def _sim_corpus(dim, n=2000, seed=0):
    rng = np.random.default_rng(seed + dim)
    rows = rng.uniform(-1, 1, (n, dim)).astype(np.float16)
    q = rng.uniform(-1, 1, dim).astype(np.float16)
    X, y = rows.astype(np.float64), q.astype(np.float64)
    e, mag = exact_distances(X, y, IP)
    e_of = np.concatenate([[np.nan], e])  # label = row + 1
    b_of = np.concatenate([[np.nan], bound_cuda_core(e, mag, dim)])
    return X, y, e_of, b_of


def _sim_lanes(X, y, dim, group_half=False):
    """DistTile16 in numpy, IP: 32 lanes, each an fma chain over its 16-byte vectors (fp32 accumulator, exact products),
    a scalar tail, then a pairwise tree over the lanes.  group_half: each 8-element group summed in fp16 first."""
    n = X.shape[0]
    acc = np.zeros((n, 32), dtype=np.float32)
    nvec = dim // 8
    for lane in range(32):
        for vi in range(lane, nvec, 32):
            if group_half:
                g = np.zeros(n, dtype=np.float16)
                for j in range(8):
                    g = (g.astype(np.float64) + X[:, 8 * vi + j] * y[8 * vi + j]).astype(np.float16)
                acc[:, lane] = (acc[:, lane].astype(np.float64) + g.astype(np.float64)).astype(np.float32)
            else:
                for j in range(8):
                    acc[:, lane] = (acc[:, lane].astype(np.float64) + X[:, 8 * vi + j] * y[8 * vi + j]).astype(np.float32)
    for el in range(8 * nvec, dim):
        lane = el - 8 * nvec
        acc[:, lane] = (acc[:, lane].astype(np.float64) + X[:, el] * y[el]).astype(np.float32)
    w = 32
    while w > 1:
        w //= 2
        acc = (acc[:, :w] + acc[:, w:2 * w]).astype(np.float32)
    return (np.float32(1.0) - acc[:, 0]).astype(np.float32)


def _select(scores32, k):
    labels = np.arange(1, len(scores32) + 1)
    order = np.lexsort((labels, scores32))[:k]
    return labels[order], scores32[order].astype(np.float64)


@pytest.mark.parametrize("dim", [128, 768, 100])
def test_checker_accepts_a_faithful_fp32_kernel(dim):
    X, y, e_of, b_of = _sim_corpus(dim)
    s = _sim_lanes(X, y, dim)
    for k in (1, 10, 129):
        labels, scores = _select(s, k)
        r = check_answer(labels, scores, e_of, b_of, k)
        assert r <= 1.0
    # the bound holds on every row, not only on the returned ones, and is not loose by orders of magnitude
    ratio = np.abs(s - e_of[1:]) / b_of[1:]
    assert ratio.max() <= 1.0 and ratio.max() > 1e-3, ratio.max()


@pytest.mark.parametrize("dim", [128, 768])
def test_checker_rejects_fp16_accumulation(dim):
    X, y, e_of, b_of = _sim_corpus(dim)
    labels, scores = _select(_sim_lanes(X, y, dim, group_half=True), 10)
    with pytest.raises(AssertionError, match="score outside the bound"):
        check_answer(labels, scores, e_of, b_of, 10)


def _gap_k(e_of, b_of):
    """The first k >= 8 whose k-th / (k+1)-th exact distances are more than 4 B apart."""
    order = np.argsort(e_of[1:]) + 1
    for k in range(8, 60):
        if e_of[order[k]] - e_of[order[k - 1]] > 4 * max(b_of[order[:k + 1]]):
            return k, order
    raise AssertionError("no gap")


@pytest.mark.parametrize("dim", [128, 768])
def test_checker_rejects_the_k_plus_first_row(dim):
    X, y, e_of, b_of = _sim_corpus(dim)
    k, order = _gap_k(e_of, b_of)
    good = order[:k]
    check_answer(good, e_of[good].astype(np.float32).astype(np.float64), e_of, b_of, k)
    wrong = np.concatenate([order[:k - 1], order[k:k + 1]])
    with pytest.raises(AssertionError, match="clearly outside"):
        check_answer(wrong, e_of[wrong].astype(np.float32).astype(np.float64), e_of, b_of, k)


@pytest.mark.parametrize("dim", [128, 768])
def test_checker_rejects_a_label_swapped_under_a_right_score_list(dim):
    X, y, e_of, b_of = _sim_corpus(dim)
    k, order = _gap_k(e_of, b_of)
    labels = order[:k].copy()
    scores = e_of[labels].astype(np.float32).astype(np.float64)
    labels[k // 2] = order[k]  # the nearest non-member, the score list untouched
    with pytest.raises(AssertionError, match="score outside the bound"):
        check_answer(labels, scores, e_of, b_of, k)


def test_checker_rejects_ties_out_of_label_order_and_short_answers():
    X, y, e_of, b_of = _sim_corpus(128)
    e_of = e_of.copy()
    order = np.argsort(e_of[1:]) + 1
    e_of[order[3]] = e_of[order[6]] = np.float32(e_of[order[3]])  # two labels of the top 20 tie exactly
    labels = np.lexsort((np.arange(1, len(e_of)), e_of[1:]))[:20] + 1
    scores = e_of[labels].astype(np.float32).astype(np.float64)
    check_answer(labels, scores, e_of, b_of, 20)
    a, b = int(np.flatnonzero(labels == order[3])[0]), int(np.flatnonzero(labels == order[6])[0])
    bad = labels.copy()
    bad[a], bad[b] = bad[b], bad[a]
    with pytest.raises(AssertionError, match="label order"):
        check_answer(bad, scores, e_of, b_of, 20)
    with pytest.raises(AssertionError):
        check_answer(labels[:19], scores[:19], e_of, b_of, 20)


def test_numpy_conversions_equal_the_oracle_conversions():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.standard_normal(3000).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, 3000).astype(np.float32),
                        np.array([0.0, -0.0, np.inf, -np.inf, 65504.0, 65519.0, 65520.0, 1e-8, 3e38], dtype=np.float32)])
    for vt in (F16, BF16):
        assert to16(x, vt).tolist() == ol.to_type(x, vt).tolist()


def test_bounds_have_the_documented_size():
    assert [chain_length(d) for d in (1, 7, 8, 9, 256, 257, 768, 771)] == [1, 1, 8, 9, 8, 9, 24, 25]
    assert 1.5e-6 < bound_cuda_core(0.0, 1.0, 768) < 2.5e-6
    assert bound_tensor_core(0.0, 1.0, 768) == 768 * 2.0 ** -22


def test_reference_fold_keeps_only_a_nan_in_the_last_row():
    nan = float("nan")
    assert reference_fold([1.0, 2.0]) == 1.0
    assert np.isnan(reference_fold([1.0, nan]))
    assert reference_fold([nan, 1.0, 2.0]) == 1.0
    assert reference_fold([3.0, nan, 2.0]) == 2.0 and reference_fold([1.0, nan, 2.0]) == 2.0
    assert reference_fold([]) == np.inf


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _vs():
    from redisearch_b200 import vecsim

    return vecsim


def _report(what, ratio):
    print(f"\n[err/B] {what}: {ratio:.4g}")


def new_index(vtype, dim, metric, rows, labels=None, multi=False):
    g = _vs().VecSimIndex(VT[vtype], dim, MT[metric], multi=multi)
    if labels is None:
        assert g.add_many(rows, label0=1) == len(rows)
    else:
        assert g.add_many(rows, labels=labels) == len(rows)
    return g


def stored_rows(g, n):
    out = np.empty((n, g.dim), dtype=np.uint16)
    assert g.L.VecSimB200_ReadRows(g.h, 0, n, out.ctypes.data) == 0
    return out


def stored_query(g, q):
    """The query as the index stores it: the library's own normaliser for cosine, bit-equal to the oracle's."""
    size = g.L.VecSimParams_GetQueryBlobSize(g.vtype, g.dim, g.metric)
    b = np.zeros(size, dtype=np.uint8)
    b[:q.nbytes] = np.ascontiguousarray(q).view(np.uint8)
    if g.metric == MT[COS]:
        o = np.ascontiguousarray(q, dtype=np.uint16).copy()
        ol.port().orc_normalize(ol._p(o), g.dim, {3: F16, 2: BF16}[g.vtype])
        _vs().normalize(b, g.dim, g.vtype)
        assert b[:q.nbytes].tobytes() == o.tobytes()
    return b


def exact_of(g, X, q, vtype, metric, n, bound):
    """e_of / b_of arrays indexed by label (= row + 1) for one query."""
    y = decode16(stored_query(g, q).view(np.uint16)[:g.dim], vtype)
    e, mag = exact_distances(X, y, metric)
    e_of = np.concatenate([[np.nan], e])
    b_of = np.concatenate([[np.nan], bound(e, mag, g.dim)])
    return e_of, b_of


def selection(S, k, allowed=None):
    """(labels, score bits) of the (score, label) selection over S (float32 scores indexed by label; NaN never selected)."""
    labels = np.arange(len(S))
    ok = ~np.isnan(S)
    if allowed is not None:
        ok &= allowed
    labels, s = labels[ok], S[ok]
    order = np.lexsort((labels, s))[:k]
    return labels[order], s[order]


def same_float(a, b):
    """Equal float32 bits, or both NaN (NaN payloads differ between the host and device folds and carry no meaning)."""
    a, b = np.float32(a), np.float32(b)
    return (np.isnan(a) and np.isnan(b)) or a.tobytes() == b.tobytes()


def assert_same_bits(labels, scores, want_labels, want_scores, what):
    assert np.asarray(labels, dtype=np.int64).tolist() == np.asarray(want_labels, dtype=np.int64).tolist(), what
    assert np.asarray(scores).astype(np.float32).tobytes() == np.asarray(want_scores, dtype=np.float32).tobytes(), what


def single_scan_scores(g, q, n):
    """Every label's score from one call (the ad-hoc context: gather_kernel over all rows), float32 indexed by label."""
    d = g.adhoc_distances(q, np.arange(1, n + 1, dtype=np.uint64))
    return np.concatenate([[np.nan], d]).astype(np.float32)


def device_batch(g, qs_stored, k):
    import torch

    nq = qs_stored.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qs_stored).view(np.int16)).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert _vs().lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    return out_l.cpu().numpy(), out_s.cpu().numpy().astype(np.float64)


def route_batch(g, qs, k, host_too=False):
    """One batch through the device API (stored-form queries), which keeps per-query flags: (labels, scores, flags).
    host_too: the host API must give the same answer."""
    stored = np.stack([stored_query(g, q).view(np.uint16)[:g.dim] for q in qs])
    labels, scores = device_batch(g, stored, k)
    flags = flags_of(g, len(qs))
    if host_too:
        hl, hs, rc = g.topk_batch(qs, k)
        assert rc == 0
        ok = hl != SIZE_MAX
        assert (labels[ok] == hl[ok].astype(np.int64)).all() and scores[ok].astype(np.float32).tobytes() == hs[ok].astype(np.float32).tobytes()
    return labels, scores, flags


def flags_of(g, nq):
    """Per-query flags of the last batch (0 exact scan, 1 / 2 the route's first / second tier, 3 label-aware exact scan);
    None where the batch keeps none (the single pass with adaptive lists)."""
    f = np.zeros(nq, dtype=np.uint32)
    return f if g.L.VecSimB200_LastCoarseFlags(g.h, f.ctypes.data, nq) == 0 else None


# ------------------------------------------------------------------------------------------------------------------
# GPU: the CUDA-core paths — one set of bits for every path, within B_cc of the exact distance
# ------------------------------------------------------------------------------------------------------------------
def _cuda_core_corpus(vtype, dim, n, seed):
    rows = ol.synth_rows(vtype, seed, 0, n, dim)
    rows[n // 2:n // 2 + 40] = rows[10:50]  # exact duplicates: ties that must resolve by label
    return rows


def _check_every_cuda_core_path(g, vtype, metric, rows, qs, ks, tag):
    """All CUDA-core paths of a single-value index on the queries qs; returns the largest err / B."""
    vs = _vs()
    n, dim = rows.shape
    X = decode16(stored_rows(g, n), vtype)
    worst = 0.0
    S_all = []
    for j, q in enumerate(qs):
        S = single_scan_scores(g, q, n)
        S_all.append(S)
        e_of, b_of = exact_of(g, X, q, vtype, metric, n, bound_cuda_core)
        # every row, not only the returned ones, within the bound
        r = np.abs(S[1:].astype(np.float64) - e_of[1:]) / b_of[1:]
        assert (r <= 1.0).all(), (tag, j, int(np.argmax(r)) + 1, r.max())
        worst = max(worst, float(r.max()))
        if j >= 2:
            continue
        qb = stored_query(g, q)
        # the batch iterator (scan_scores_kernel): the full (score, label) order, in chunks
        want_l, want_s = selection(S, n)
        it = g.batch_iterator(q)
        got_l, got_s = [], []
        while it.has_next():
            ids, sc, code = it.next(347, vs.BY_SCORE)
            assert code == 0
            if not len(ids):
                break
            got_l += ids.tolist()
            got_s += sc.tolist()
        it.free()
        assert_same_bits(got_l, got_s, want_l, want_s, (tag, j, "batch iterator"))
        for k in ks:  # the single query (scan_topk, fused and unfused)
            gi, gs, code = g.topk(q, k)
            assert code == 0
            wl, ws = selection(S, k)
            assert_same_bits(gi, gs, wl, ws, (tag, j, k, "TopKQuery"))
            worst = max(worst, check_answer(gi, gs, e_of, b_of, k))
        # filtered KNN over all labels and over every third label (gather_kernel)
        for allowed in (None, np.arange(n + 1) % 3 == 1):
            ids = np.arange(1, n + 1, dtype=np.uint32) if allowed is None else np.flatnonzero(allowed).astype(np.uint32)
            fl, fs, rc = g.topk_filtered(q, 10, ids)
            assert rc == 0
            wl, ws = selection(S, 10, allowed)
            assert_same_bits(fl, fs, wl, ws, (tag, j, "TopKFiltered"))
        # GetDistanceFrom on the stored query: the tied duplicates, the nearest rows, a few others
        for lab in [11, 12, n // 2 + 1, n // 2 + 2, 1, n] + want_l[:5].tolist():
            d = g.distance_from(int(lab), qb)
            assert np.float32(d).tobytes() == S[lab].tobytes(), (tag, j, lab, d, S[lab])
        assert np.isnan(g.distance_from(n + 7, qb))
        # the range query: exactly the rows whose single-scan score is <= (float)radius
        for pos in (0, 9, 37):
            radius = max(0.0, float(want_s[min(pos, n - 1)]))  # inner-product distances can be negative; radii cannot
            ri, rs, code = g.range(q, radius)
            assert code == 0
            inside = ~np.isnan(S) & (S <= np.float32(radius))
            assert sorted(ri.tolist()) == np.flatnonzero(inside).tolist(), (tag, j, pos)
            assert rs.astype(np.float32).tobytes() == S[ri].tobytes()
            assert (np.diff(rs) >= 0).all()
    # batches on the exact scan: QT = 8 query tiles and the partial tiles
    vs.lib().VecSimB200_SetCoarseMode(0)
    try:
        Q = np.ascontiguousarray(qs)
        for nq, ks_b in ((1, (10,)), (3, (10,)), (9, (1, 10)), (15, (10, 128, 129))):
            for k in ks_b:
                bl, bs, rc = g.topk_batch(Q[:nq], k)
                assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 0
                for i in range(nq):
                    h = int((bl[i] != SIZE_MAX).sum())
                    wl, ws = selection(S_all[i], k)
                    assert_same_bits(bl[i, :h], bs[i, :h], wl, ws, (tag, nq, k, i, "TopKQueryBatch"))
        radii = np.array([max(0.0, float(selection(S_all[i], 20)[1][-1])) for i in range(9)])
        replies, rc, flags = g.range_batch(Q[:9], radii)
        assert rc == 0
        for i, (ri, rs, code) in enumerate(replies):
            inside = ~np.isnan(S_all[i]) & (S_all[i] <= np.float32(radii[i]))
            assert code == 0 and sorted(ri.tolist()) == np.flatnonzero(inside).tolist(), (tag, i, "RangeQueryBatch")
            assert rs.astype(np.float32).tobytes() == S_all[i][ri].tobytes()
    finally:
        vs.lib().VecSimB200_SetCoarseMode(-1)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP, COS])
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_cuda_core_paths_over_dim_residuals(vtype, metric):
    worst = 0.0
    for dim in DIM_SWEEP:
        n = 1200
        rows = _cuda_core_corpus(vtype, dim, n, 500 + dim)
        g = new_index(vtype, dim, metric, rows)
        qs = ol.synth_rows(vtype, 900 + dim, 0, 15, dim)
        qs[1] = rows[13]  # its best rows include a tied pair (cosine / L2)
        worst = max(worst, _check_every_cuda_core_path(g, vtype, metric, rows, qs, (1, 10, 128, 129, 1000), (dim,)))
        g.close()
    _report(f"CUDA-core paths {TNAME[vtype]} {MNAME[metric]} (dims {DIM_SWEEP[0]}..{DIM_SWEEP[-1]})", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric,n,dim", [(F16, L2, 70_000, 128), (BF16, IP, 70_000, 100), (F16, COS, 20_000, 128),
                                                (BF16, L2, 66_000, 776)])
def test_batches_the_tensor_cores_do_not_take(vtype, metric, n, dim):
    """L2 at any batch size, dim % 8 != 0, n < 65,536: the default mode answers these batches with the exact scan."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(-1)
    rows = ol.synth_rows(vtype, 61, 0, n, dim)
    g = new_index(vtype, dim, metric, rows)
    X = decode16(stored_rows(g, n), vtype)
    qs = ol.synth_rows(vtype, 62, 0, 40, dim)
    worst = 0.0
    for nq, k in ((40, 10), (16, 128)):
        bl, bs, rc = g.topk_batch(qs[:nq], k)
        assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 0
        for i in range(0, nq, 3):
            S = single_scan_scores(g, qs[i], n)
            wl, ws = selection(S, k)
            assert_same_bits(bl[i], bs[i], wl, ws, (nq, k, i))
            e_of, b_of = exact_of(g, X, qs[i], vtype, metric, n, bound_cuda_core)
            worst = max(worst, check_answer(bl[i].astype(np.int64), bs[i], e_of, b_of, k))
    _report(f"exact-scan batches {TNAME[vtype]} {MNAME[metric]} n={n} dim={dim}", worst)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the direct 16-bit tensor-core route
# ------------------------------------------------------------------------------------------------------------------
WGMMA_MAX_DIM = 1024  # coarse_tc.cu wgmma_fits: the queries' 2 * dim bytes (16 K blocks) and two ring stages in 227 KB


def _exact_many(g, X_bits, qs, vtype, metric, bound):
    """e_of / b_of [nq][n + 1] for many queries (inner product / cosine), in row chunks."""
    n, dim = X_bits.shape
    Y = np.stack([decode16(stored_query(g, q).view(np.uint16)[:dim], vtype) for q in qs])
    dot = np.empty((len(qs), n))
    mag = np.empty((len(qs), n))
    for r0 in range(0, n, 8192):
        Xc = decode16(X_bits[r0:r0 + 8192], vtype)
        dot[:, r0:r0 + 8192] = Y @ Xc.T
        mag[:, r0:r0 + 8192] = np.abs(Y) @ np.abs(Xc).T
    e = 1.0 - dot
    nanc = np.full((len(qs), 1), np.nan)
    return np.hstack([nanc, e]), np.hstack([nanc, bound(e, mag, dim)])


def _tc_case(vtype, metric, dim, n, batches, seed=42, rows=None, qs=None, want_path=2):
    """Batches (nq, k) on the tensor-core route, every answered query checked against B_tc; returns (max err / B, flags)."""
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(-1)
    if rows is None:
        rows = ol.synth_rows(vtype, seed, 0, n, dim)
    g = new_index(vtype, dim, metric, rows)
    if qs is None:
        qs = ol.synth_rows(vtype, seed + 1, 0, max(nq for nq, _ in batches), dim)
    checked = sorted({i for nq, _ in batches for i in (range(nq) if nq <= 40 else range(0, nq, 4))})
    e_all, b_all = _exact_many(g, stored_rows(g, n), qs[checked], vtype, metric, bound_tensor_core)
    row_of = {q: j for j, q in enumerate(checked)}
    worst, seen = 0.0, []
    for b, (nq, k) in enumerate(batches):
        bl, bs, f = route_batch(g, qs[:nq], k, host_too=b == 0)
        assert vs.lib().VecSimB200_LastBatchPath(g.h) == want_path, (dim, nq, k)
        seen += f.tolist() if f is not None else [4] * nq  # 4: the batch keeps no flags (VECSIM_B200_FIXED=0)
        for i in range(nq):
            if i in row_of:
                j = row_of[i]
                worst = max(worst, check_answer(bl[i].astype(np.int64), bs[i], e_all[j], b_all[j], k))
    g.close()
    return worst, np.bincount(np.asarray(seen, dtype=np.int64), minlength=5)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [IP, COS])
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_direct_tensor_core_route_within_its_bound(vtype, metric):
    worst_all = 0.0
    for dim in (32, 40, 128, 768, 776, WGMMA_MAX_DIM):
        worst, flags = _tc_case(vtype, metric, dim, 66_000, ((16, 1), (40, 10), (256, 100), (16, 128)), seed=7 + dim)
        assert flags[1] + flags[2] == flags.sum(), flags.tolist()  # every query is answered on the route (tier 1 or 2)
        _report(f"tensor-core route {TNAME[vtype]} {MNAME[metric]} dim={dim} (flags tier1/tier2 {flags[1]}/{flags[2]})", worst)
        worst_all = max(worst_all, worst)
    _report(f"tensor-core route {TNAME[vtype]} {MNAME[metric]}, all dims", worst_all)
    # one dimension past the shared-memory limit leaves the route (and the bound of the exact scan applies)
    rows = ol.synth_rows(vtype, 3, 0, 66_000, WGMMA_MAX_DIM + 8)
    g = new_index(vtype, WGMMA_MAX_DIM + 8, metric, rows)
    assert g.topk_batch(ol.synth_rows(vtype, 4, 0, 16, WGMMA_MAX_DIM + 8), 10)[2] == 0
    assert _vs().lib().VecSimB200_LastBatchPath(g.h) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("env", ["VECSIM_B200_FIXED=0", "VECSIM_B200_TIER2=0"])
def test_direct_route_variants_within_the_bound(env):
    """The single pass with adaptive lists (VECSIM_B200_FIXED=0) and the route without its second tier (VECSIM_B200_TIER2=0)
    answer within the same bound (the switches are read once per process: checked in a subprocess)."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = (
        "import sys\n"
        f"sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})\n"
        "import test_half_precision_bounds as t\n"
        "for vt, mt, dim in ((t.F16, t.IP, 128), (t.BF16, t.COS, 776)):\n"
        "    w, f = t._tc_case(vt, mt, dim, 66_000, ((40, 10), (16, 128)))\n"
        "    assert w <= 1.0 and f[0] == 0 and f[3] == 0, (w, f)  # f[4]: no flags kept (single pass)\n"
        "    print('RATIO', dim, w, f.tolist())\n"
        "print('VARIANT-OK')\n"
    )
    name, value = env.split("=")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=dict(os.environ, **{name: value}))
    assert r.returncode == 0 and "VARIANT-OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    print("\n" + env + ": " + " | ".join(line for line in r.stdout.splitlines() if line.startswith("RATIO")))


# ------------------------------------------------------------------------------------------------------------------
# GPU: adversarial cases for the fixed-bound pass
# ------------------------------------------------------------------------------------------------------------------
def _sample_stride(n, k, nq):
    """vecsim_index.cpp batch_scan_rows: the sample pass visits every stride-th row tile of 128 rows."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = (n + 127) // 128
    grid_y = (nq + 63) // 64
    gx = max(1, min(tiles, sms // grid_y))
    f = min(0.25, max(0.01, k / (64.0 * gx)))
    return int(max(1.0, min(math.floor(1.0 / f), math.floor(tiles / (2.0 * k))))), gx


def _planted(vtype, dim, n, rng):
    """A query direction q, far rows (distance ~ 1 + |q|^2 / 2, all distinct), and the 16-bit blobs of c * q."""
    q = rng.uniform(0.25, 1.0, dim).astype(np.float32) * np.where(rng.random(dim) < 0.5, -1, 1)
    far = -0.5 * q[None, :] + 0.05 * rng.standard_normal((n, dim)).astype(np.float32)
    return q, far, lambda x: to16(x, vtype)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_fixed_bound_keeps_every_row_tied_with_it(vtype):
    """k - 1 rows strictly better than everything, bit-identical copies of the k-th best row at one offset of every row tile but
    tile 0, all other rows far.  The sample's k-th slice minimum is exactly the copy's distance, so the bound is the copy's
    distance itself and the main pass must keep every copy; the k-th answer is the copy in tile 1, a tile the sample never visits."""
    n, dim, nq, k, off = 70_000, 128, 16, 10, 77
    stride, _ = _sample_stride(n, k, nq)
    assert stride > 1
    rng = np.random.default_rng(21)
    q, far, conv = _planted(vtype, dim, n, rng)
    rows = conv(far)
    better = conv(np.stack([(0.9 - 0.02 * j) * q for j in range(k - 1)]))
    rows[:k - 1] = better  # tile 0, rows 0..k-2
    copy = conv((0.5 * q)[None, :])[0]
    rows[128 + off::128] = copy  # offset 77 of tiles 1, 2, ...
    n_copies = len(range(128 + off, n, 128))
    qs = np.repeat(conv(q[None, :]), nq, axis=0)
    g = new_index(vtype, dim, IP, rows)
    bl, bs, f = route_batch(g, qs, k, host_too=True)
    assert _vs().lib().VecSimB200_LastBatchPath(g.h) == 2
    assert (f == 1).all(), f.tolist()  # the fixed-bound tier proved every query
    e_all, b_all = _exact_many(g, stored_rows(g, n), qs[:1], vtype, IP, bound_tensor_core)
    want = list(range(1, k)) + [128 + off + 1]
    for i in range(nq):
        assert bl[i].astype(np.int64).tolist() == want, (i, bl[i].tolist())
        worst = check_answer(bl[i].astype(np.int64), bs[i], e_all[0], b_all[0], k)
    # every copy scores the same bits on the route: k = 128 returns 119 of them in row order
    bl, bs, f = route_batch(g, qs, 128)
    assert (f == 1).all(), f.tolist()
    assert bl[0, k - 1:].astype(np.int64).tolist() == [128 * t + off + 1 for t in range(1, 128 - k + 2)]
    assert len(set(bs[0, k - 1:].tolist())) == 1 and n_copies > 128
    _report(f"tensor-core ties at the bound {TNAME[vtype]}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_ties_overflowing_a_row_range_resolve_by_label_on_the_second_tier(vtype):
    """More than 256 copies of the k-th best row in one row range of the main pass (tiles t, t + gx, ...): its list overflows,
    the query goes to the second tier (flag 2), and the tie still resolves to the lowest labels."""
    n, dim, nq, k = 70_000, 128, 16, 10
    _, gx = _sample_stride(n, k, nq)
    rng = np.random.default_rng(22)
    q, far, conv = _planted(vtype, dim, n, rng)
    rows = conv(far)
    rows[:k - 1] = conv(np.stack([(0.9 - 0.02 * j) * q for j in range(k - 1)]))
    copy = conv((0.5 * q)[None, :])[0]
    tiles = [5 + j * gx for j in range(4)]
    for t in tiles:
        rows[t * 128:t * 128 + 100] = copy  # 400 copies in the row range of tile 5
    qs = np.repeat(conv(q[None, :]), nq, axis=0)
    g = new_index(vtype, dim, IP, rows)
    e_all, b_all = _exact_many(g, stored_rows(g, n), qs[:1], vtype, IP, bound_tensor_core)
    for k_ in (k, 100):
        bl, bs, f = route_batch(g, qs, k_, host_too=True)
        assert _vs().lib().VecSimB200_LastBatchPath(g.h) == 2
        assert (f == 2).all(), f.tolist()
        want = list(range(1, k)) + [t * 128 + j + 1 for t in tiles for j in range(100)][:k_ - k + 1]
        for i in range(nq):
            assert bl[i].astype(np.int64).tolist() == want, (k_, i, bl[i][:12].tolist())
            worst = check_answer(bl[i].astype(np.int64), bs[i], e_all[0], b_all[0], k_)
    _report(f"tensor-core ties on the second tier {TNAME[vtype]}", worst)


@pytest.mark.gpu
def test_clustered_corpus_overflowing_a_row_range_reaches_the_second_tier():
    """Clusters of near-duplicates, as in test_vecsim_coarse.py's clustered corpus, but 300 of them per query, in three row tiles
    of one row range of the main pass that the sample pass does not visit: more rows fall below the bound than that range's list
    of 256 holds, so every query of an odd-sized batch (nq = 17, k = 7) is gathered into the second tier (flag 2)."""
    vtype, n, dim, nq, k = F16, 70_000, 128, 17, 7
    stride, gx = _sample_stride(n, k, nq)
    bases = [b for b in range(1, gx) if all((b + j * gx) % stride for j in range(3))][:nq]
    assert len(bases) == nq and (bases[-1] + 2 * gx + 1) * 128 <= n
    rng = np.random.default_rng(23)
    rows = ol.synth_rows(vtype, 31, 0, n, dim)
    centers = rng.uniform(-1, 1, (nq, dim)).astype(np.float32)
    for b, center in zip(bases, centers):
        for t in (b, b + gx, b + 2 * gx):
            rows[t * 128:t * 128 + 100] = to16(center[None, :] + 2e-3 * rng.standard_normal((100, dim)).astype(np.float32), vtype)
    qs = to16(centers + 2e-3 * rng.standard_normal((nq, dim)).astype(np.float32), vtype)
    g = new_index(vtype, dim, COS, rows)
    bl, bs, f = route_batch(g, qs, k, host_too=True)
    assert _vs().lib().VecSimB200_LastBatchPath(g.h) == 2
    assert f is not None and (f == 2).all(), f
    e_all, b_all = _exact_many(g, stored_rows(g, n), qs, vtype, COS, bound_tensor_core)
    worst = 0.0
    for i in range(nq):
        worst = max(worst, check_answer(bl[i].astype(np.int64), bs[i], e_all[i], b_all[i], k))
    _report(f"tensor-core clustered corpus on the second tier {TNAME[vtype]}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_duplicates_across_the_k_boundary_on_the_route(vtype):
    """Exact duplicates of rows (as the 8-bit route's test plants them) and a query equal to one of them: ties at every k
    resolve to the lower label, on the route and on the exact scan alike."""
    vs = _vs()
    n, dim, nq = 70_000, 128, 40
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    rows[5000:5040] = rows[4000:4040]
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[1] = rows[4003]
    g = new_index(vtype, dim, COS, rows)
    e_all, b_all = _exact_many(g, stored_rows(g, n), qs[:4], vtype, COS, bound_tensor_core)
    for k in (1, 2, 10, 128):
        bl, bs, rc = g.topk_batch(qs, k)
        assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 2
        for i in range(4):
            check_answer(bl[i].astype(np.int64), bs[i], e_all[i], b_all[i], k)
        # the two copies sit at different offsets of their row tiles: the route owes them equal bits only within its bound
        assert set(bl[1, :2].tolist()) <= {4004, 5004} and (k == 1 or set(bl[1, :2].tolist()) == {4004, 5004}), bl[1, :3]
    S = single_scan_scores(g, qs[1], n)
    assert S[4004] == S[5004]
    for k in (1, 2, 3):
        gi, gs, _ = g.topk(qs[1], k)
        assert_same_bits(gi, gs, *selection(S, k), "single query")


# ------------------------------------------------------------------------------------------------------------------
# GPU: dynamic range
# ------------------------------------------------------------------------------------------------------------------
def _fp16_with_subnormals(rng, n, dim, frac):
    x = rng.uniform(-1, 1, (n, dim)).astype(np.float16)
    sub = rng.random((n, dim)) < frac
    x[sub] = (rng.integers(1, 1024, int(sub.sum())) * np.where(rng.random(int(sub.sum())) < 0.5, -1, 1)).astype(np.float64) * 2.0 ** -24
    return x.view(np.uint16)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [L2, IP])
def test_fp16_subnormal_and_largest_values_on_the_cuda_cores(metric):
    rng = np.random.default_rng(31)
    n, dim = 1200, 72
    rows = _fp16_with_subnormals(rng, n, dim, 0.6)
    rows[100:200] = _fp16_with_subnormals(rng, 100, dim, 1.0)  # rows with only subnormal components
    big = rng.uniform(-65504, 65504, (50, dim)).astype(np.float16)
    big[:, :3] = np.float16(65504.0)
    rows[300:350] = big.view(np.uint16)
    qs = _fp16_with_subnormals(rng, 15, dim, 0.6)
    qs[2] = _fp16_with_subnormals(rng, 1, dim, 1.0)[0]
    qs[3] = rows[301]
    g = new_index(F16, dim, metric, rows)
    worst = _check_every_cuda_core_path(g, F16, metric, rows, qs, (1, 10, 129), ("subnormal",))
    _report(f"CUDA-core paths fp16 {MNAME[metric]} subnormal / 65504", worst)


@pytest.mark.gpu
def test_fp16_subnormal_and_largest_values_on_the_route():
    rng = np.random.default_rng(32)
    n, dim = 66_000, 128
    rows = _fp16_with_subnormals(rng, n, dim, 0.5)
    rows[1000:3000] = _fp16_with_subnormals(rng, 2000, dim, 1.0)
    rows[5000:5050, :4] = np.float16(65504.0).view(np.uint16)
    qs = _fp16_with_subnormals(rng, 40, dim, 0.5)
    qs[:8] = _fp16_with_subnormals(rng, 8, dim, 1.0)  # queries with only subnormal components
    worst, flags = _tc_case(F16, IP, dim, n, ((16, 10), (40, 128)), rows=rows, qs=qs)
    assert flags[1] + flags[2] == flags.sum(), flags.tolist()
    _report("tensor-core route fp16 IP subnormal / 65504", worst)


def _bf16_wide(rng, n, dim):
    """bf16 rows of moderate size, rows whose products sum to ~1e37 (finite in fp32), and rows whose same-sign products
    overflow fp32 (+inf dot -> -inf distance; -inf dot -> +inf distance)."""
    rows = ol.synth_rows(BF16, 77, 0, n, dim)
    rows[200:220] = to16(np.full((20, dim), 1.0e36, dtype=np.float32) * rng.uniform(0.5, 1, (20, dim)).astype(np.float32), BF16)
    rows[400:410] = to16(np.full((10, dim), 1.0e38, dtype=np.float32), BF16)
    rows[600:605] = to16(np.full((5, dim), -1.0e38, dtype=np.float32), BF16)
    q = to16(rng.uniform(0.5, 1.0, (16, dim)).astype(np.float32), BF16)
    return rows, q


def _overflow_expectation(g, rows, qs, vtype, metric, bound):
    """e_of / b_of from the stored values, with the labels whose fp32 sum overflows set to what the reference's
    fp32-accumulate tier returns for them (the C restatement, AVX-512 tier)."""
    n, dim = rows.shape
    p = ol.PortIndex(vtype, dim, metric, tier=ol.TIER_AVX512)
    p.add_many(rows, 1)
    X = decode16(stored_rows(g, n), vtype)
    out = []
    for q in qs:
        e_of, b_of = exact_of(g, X, q, vtype, metric, n, bound)
        over = np.flatnonzero(np.abs(1.0 - e_of[1:]) > 3.0e38) + 1
        for lab in over.tolist():
            e_of[lab] = p.distance_from(lab, stored_query(g, q))
            assert np.isinf(e_of[lab]), (lab, e_of[lab])
        assert len(over) == 15
        out.append((e_of, b_of))
    return out


@pytest.mark.gpu
def test_bf16_wide_magnitudes_and_fp32_overflow():
    vs = _vs()
    rng = np.random.default_rng(33)
    # CUDA-core paths
    n, dim = 1200, 64
    rows, qs = _bf16_wide(rng, n, dim)
    g = new_index(BF16, dim, IP, rows)
    exp = _overflow_expectation(g, rows, qs[:2], BF16, IP, bound_cuda_core)
    worst = 0.0
    for j in range(2):
        S = single_scan_scores(g, qs[j], n)
        for k in (1, 10, 40):
            gi, gs, _ = g.topk(qs[j], k)
            assert_same_bits(gi, gs, *selection(S, k), (j, k))
            worst = max(worst, check_answer(gi, gs, exp[j][0], exp[j][1], k))
        gi, gs, _ = g.topk(qs[j], n)
        assert (gs[:10] == -np.inf).all() and (gs[-5:] == np.inf).all()
        assert gi[:10].tolist() == list(range(401, 411))
    _report("CUDA-core paths bf16 IP wide magnitudes", worst)
    # the route
    n = 66_000
    rows, qs = _bf16_wide(rng, n, dim)
    g = new_index(BF16, dim, IP, rows)
    exp = _overflow_expectation(g, rows, qs[:4], BF16, IP, bound_tensor_core)
    worst = 0.0
    for k in (5, 10, 40, 128):
        bl, bs, rc = g.topk_batch(qs, k)
        assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 2
        for i in range(4):
            worst = max(worst, check_answer(bl[i].astype(np.int64), bs[i], exp[i][0], exp[i][1], k))
            assert bl[i, :min(k, 10)].astype(np.int64).tolist() == list(range(401, 401 + min(k, 10)))
    _report("tensor-core route bf16 IP wide magnitudes", worst)


# ------------------------------------------------------------------------------------------------------------------
# GPU: multi-value indexes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(F16, IP), (BF16, COS)])
def test_multi_value_batches_against_the_per_label_minimum(vtype, metric):
    """16-bit multi-value batches: the label-aware route (flags 1 / 2, B_tc) and the label-aware exact scan it falls back to
    (flag 3, B_cc), against the float64 minimum over each label's rows."""
    vs = _vs()
    rng = np.random.default_rng(41)
    cases = []
    n, dim = 70_000, 128
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    cases.append(("3 rows per label", rows, (np.arange(n) // 3 + 1).astype(np.uint64), ol.synth_rows(vtype, 43, 0, 40, dim)))
    dim2, n_labels = 64, 1600
    centres = rng.uniform(-0.7, 0.7, (n_labels, dim2)).astype(np.float32)
    x = np.repeat(centres, 50, axis=0) + 0.02 * rng.standard_normal((n_labels * 50, dim2)).astype(np.float32)
    qx = centres[rng.integers(0, n_labels, 32)] + 0.02 * rng.standard_normal((32, dim2)).astype(np.float32)
    conv = lambda a: to16(a, vtype)  # noqa: E731
    cases.append(("50-row chunks", conv(x), np.repeat(1 + np.arange(n_labels, dtype=np.uint64), 50), conv(qx)))
    for name, rows, labels, qs in cases:
        n, d = rows.shape
        g = new_index(vtype, d, metric, rows, labels=labels, multi=True)
        bits = stored_rows(g, n)
        row_labels = labels.astype(np.int64)
        for k in (10, 100):
            bl, bs, f = route_batch(g, qs, k, host_too=True)
            assert vs.lib().VecSimB200_LastBatchPath(g.h) == 2 and f is not None
            worst = {1: 0.0, 3: 0.0}
            for i in range(0, len(qs), 2):
                route = f[i] in (1, 2)
                bound = bound_tensor_core if route else bound_cuda_core
                y = decode16(stored_query(g, qs[i]).view(np.uint16)[:d], vtype)
                e_r, m_r = exact_distances(decode16(bits, vtype), y, metric)
                e_of, b_of = per_label(e_r, bound(e_r, m_r, d), row_labels, int(labels.max()) + 1)
                h = int((bl[i] >= 0).sum())
                r = check_answer(bl[i, :h].astype(np.int64), bs[i, :h], e_of, b_of, k)
                worst[1 if route else 3] = max(worst[1 if route else 3], r)
            _report(f"multi-value {name} {TNAME[vtype]} {MNAME[metric]} k={k} flags {np.bincount(f, minlength=4).tolist()}: "
                    f"route {worst[1]:.4g}, label-aware exact scan", worst[3])
            if name == "50-row chunks":
                assert (f == 3).sum() >= len(qs) // 2
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("vtype,metric", [(F16, L2), (BF16, IP), (F16, COS)])
def test_multi_value_filtered_knn_and_distances(vtype, metric):
    """TopKFiltered on a multi-value index (gather_min_kernel) within B_cc of the per-label minimum, and GetDistanceFrom / the
    ad-hoc context bit-equal to it on every label."""
    rng = np.random.default_rng(42)
    n, dim = 3000, 40
    rows = ol.synth_rows(vtype, 45, 0, n, dim)
    labels = rng.integers(1, 601, n).astype(np.uint64)  # 600 labels, rows interleaved
    g = new_index(vtype, dim, metric, rows, labels=labels, multi=True)
    X = decode16(stored_rows(g, n), vtype)
    worst = 0.0
    for q in ol.synth_rows(vtype, 46, 0, 3, dim):
        y = decode16(stored_query(g, q).view(np.uint16)[:dim], vtype)
        e_r, m_r = exact_distances(X, y, metric)
        e_of, b_of = per_label(e_r, bound_cuda_core(e_r, m_r, dim), labels.astype(np.int64), 601)
        present = np.flatnonzero(~np.isnan(e_of))
        for k in (1, 10, 128):
            fl, fs, rc = g.topk_filtered(q, k, present.astype(np.uint32))
            assert rc == 0
            worst = max(worst, check_answer(fl.astype(np.int64), fs, e_of, b_of, k, tie_order=False))
        qb = stored_query(g, q)
        adhoc = g.adhoc_distances(q, present.astype(np.uint64))
        for lab, a in zip(present.tolist(), adhoc.tolist()):
            fl, fs, rc = g.topk_filtered(q, 1, np.array([lab], dtype=np.uint32))
            assert rc == 0 and fl.tolist() == [lab]
            d = g.distance_from(lab, qb)
            assert np.float32(d).tobytes() == np.float32(fs[0]).tobytes() == np.float32(a).tobytes(), (lab, d, fs[0], a)
    _report(f"multi-value filtered KNN {TNAME[vtype]} {MNAME[metric]}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [F16, BF16])
def test_multi_value_distance_folds_nan_like_the_reference(vtype):
    """A NaN row (inf * 0) first, in the middle and last among a label's rows: GetDistanceFrom, the ad-hoc context and
    TopKFiltered all give the reference's float fold, where only a NaN in the last row survives.  An unknown label is NaN."""
    dim = 8
    inf = np.float32(np.inf)
    q32 = np.array([0, 1, 1, 1, 1, 1, 1, 1], dtype=np.float32)
    nan_row = np.array([inf, 0, 0, 0, 0, 0, 0, 0], dtype=np.float32)  # inf * 0 = NaN in the dot product

    def row(c):
        return np.full(dim, c, dtype=np.float32) * np.array([0, 1, 1, 1, 1, 1, 1, 1], dtype=np.float32)

    # label -> its rows in insertion order; small integers: every distance is exact in fp32
    groups = {1: [nan_row, row(0.5), row(1.0)], 2: [row(1.0), nan_row, row(0.25)], 3: [row(0.5), row(0.25), nan_row],
              4: [row(2.0), row(1.0)], 5: [nan_row], 6: [row(0.75)]}
    conv = lambda a: to16(a, vtype)  # noqa: E731
    g = _vs().VecSimIndex(VT[vtype], dim, MT[IP], multi=True)
    ref = ol.RefIndex(vtype, dim, IP, multi=True) if ol.ref_vecsim() is not None else None
    for lab, rs in groups.items():
        for r in rs:
            assert g.add(conv(r[None, :])[0], lab) == 1
            if ref is not None:
                ref.add(conv(r[None, :])[0], lab)
    q = conv(q32[None, :])[0]
    qb = stored_query(g, q)
    want = {lab: reference_fold([np.float32(1.0) - np.float32(np.dot(r[1:], q32[1:])) if not np.isinf(r[0]) else np.nan for r in rs])
            for lab, rs in groups.items()}
    # NaN first: forgotten; in the middle: the rows before it are forgotten too (a plain min gives -6); last: kept
    assert want[1] == np.float32(-6.0) and want[2] == np.float32(-0.75) and np.isnan(want[3]) and np.isnan(want[5])
    labs = np.array(sorted(groups) + [99], dtype=np.uint64)
    adhoc = g.adhoc_distances(q, labs)
    for lab, a in zip(labs.tolist(), adhoc.tolist()):
        d = g.distance_from(lab, qb)
        if lab == 99:
            assert np.isnan(d) and np.isnan(a)
            continue
        w = want[lab]
        assert same_float(d, w) and same_float(a, w), (lab, d, a, w)
        if ref is not None:
            assert same_float(ref.distance_from(lab, qb), w)
    fl, fs, rc = g.topk_filtered(q, 10, np.array(sorted(groups), dtype=np.uint32))
    assert rc == 0
    got = dict(zip(fl.tolist(), fs.tolist()))
    assert set(got) == {lab for lab in groups if not np.isnan(want[lab])}  # NaN docIds are skipped
    for lab, s in got.items():
        assert np.float32(s).tobytes() == want[lab].tobytes()
