"""GPU: the tensor-core coarse pass (csrc/coarse_tc.cu) must return EXACTLY what the exact scan returns.

wgmma GEMM (mode 1: fp16 shadow rows, mode 2: TF32 on the fp32 rows) + fused candidate lists -> exact rescoring (bit-exact arithmetic) -> per-query
completeness proof -> on-device fallback.  Whatever the proof decides, ids and scores must equal the
oracle's bit for bit; the flags tell how many queries were served by the tensor-core path.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol

pytestmark = pytest.mark.gpu


def _device_batch(vs, torch, index, qs_norm, k):
    nq = qs_norm.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qs_norm)).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = vs.lib().VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp)
    assert rc == 0
    torch.cuda.synchronize()
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)
    return out_l.cpu().numpy(), out_s.cpu().numpy(), (flags if frc == 0 else None)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n,dim,nq,k", [(70_000, 128, 40, 10), (66_000, 768, 64, 10), (131_072, 96, 17, 16), (80_000, 104, 33, 5),
                                        (70_000, 128, 128, 10), (300_000, 64, 256, 10), (66_000, 256, 512, 8),
                                        (66_000, 1024, 70, 10), (70_000, 32, 40, 10), (70_000, 40, 40, 10), (66_000, 776, 64, 10),
                                        (66_000, 1016, 64, 10), (70_000, 128, 401, 9)])
def test_coarse_path_is_exact(n, dim, nq, k, mode):
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(mode)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS)(dim)  # the reference's own compiled code when oracle/_ref is present
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None, "the batch did not take the tensor-core path"
    assert (flags != 0).sum() >= nq * 0.9, f"only {int(flags.sum())}/{nq} queries were verified by the coarse path"
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist(), (i, flags[i], labels[i], pi)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    # the host-facing batch entry point goes through the same pipeline
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and (hl.astype(np.int64) == labels).all()
    # and switching the coarse path off gives the same answer from the exact scan
    vs.lib().VecSimB200_SetCoarseMode(0)
    l2, s2, f2 = _device_batch(vs, torch, g, qn, k)
    assert f2 is None and (l2 == labels).all() and s2.tobytes() == scores.tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)


def test_shadow_rows_follow_updates_and_deletes():
    """mode 1 keeps an fp16 copy of the rows: appended rows, overwritten labels and rows moved by a
    swap-delete (brute_force.h:196-224) must reach it before the next coarse batch."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 64, 32, 10
    rows = ol.synth_rows(ol.F32, 7, 0, n + 2000, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
    g.add_many(rows[:n], label0=1)
    p.add_many(rows[:n], 1)
    qs = ol.synth_rows(ol.F32, 8, 0, nq, dim)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)

    def check():
        labels, scores, flags = _device_batch(vs, torch, g, qn, k)
        assert flags is not None and (flags != 0).sum() >= nq * 0.9
        for i in range(nq):
            pi, ps = p.topk(qs[i], k)
            assert labels[i].tolist() == pi.tolist(), (i, labels[i], pi)
            assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
        return labels

    first = check()  # builds the shadow
    # delete the current best hit of every query (swap-delete moves the last rows into the holes) ...
    for lab in sorted({int(x) for x in first[:, 0]}):
        assert g.delete(lab) == 1
        p.delete(lab)
    # ... overwrite some labels with the query vectors themselves (they become the new best hits) ...
    for i in range(0, nq, 4):
        g.add(qs[i], 1000 + i)
        p.add(qs[i], 1000 + i)
    # ... and append fresh rows
    g.add_many(rows[n:], label0=n + 1)
    p.add_many(rows[n:], n + 1)
    second = check()
    for i in range(0, nq, 4):
        assert second[i, 0] == 1000 + i
    vs.lib().VecSimB200_SetCoarseMode(-1)


def _checker(metric_code):
    """The reference's own compiled code when oracle/_ref is present, else the C restatement (pinned to it)."""
    def make(dim):
        if ol.ref_vecsim() is not None:
            return ol.RefIndex(ol.F32, dim, metric_code)
        return ol.PortIndex(ol.F32, dim, metric_code, tier=ol.TIER_AVX512)
    return make


def test_deleted_then_reused_row_ids_do_not_keep_stale_shadow_rows():
    """Delete the LAST rows (no swap, nothing marked dirty), then append rows that are the exact nearest neighbours of
    the queries: they land on the re-used row ids.  A shadow that still held the deleted rows would score those ids
    against the wrong vectors and the proof would pass on a wrong answer (round-1 advisor finding)."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 64, 32, 10
    rows = ol.synth_rows(ol.F32, 17, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS)(dim)
    g.add_many(rows, label0=1)
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 18, 0, nq, dim)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    labels, _, flags = _device_batch(vs, torch, g, qn, k)  # builds the shadow over all n rows
    assert flags is not None
    for lab in range(n, n - nq, -1):  # always the last row: removeVector does not move anything
        assert g.delete(lab) == 1
        p.delete(lab)
    for i in range(nq):  # the new rows ARE the queries: distance ~0, on the row ids just vacated
        assert g.add(qs[i], 5_000_000 + i) == 1
        p.add(qs[i], 5_000_000 + i)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i, 0] == 5_000_000 + i, (i, labels[i], pi)
        assert labels[i].tolist() == pi.tolist(), (i, flags[i], labels[i], pi)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)


def _snap_against(x, q, against):
    """x with every component just short of an fp16 rounding midpoint, on the side where round-to-nearest moves the
    dot product with q down (against) or up; x's components must lie in the fp16 normal range."""
    ax = np.abs(x.astype(np.float64))
    ulp = 2.0 ** (np.floor(np.log2(ax)) - 10)
    lo = np.floor(ax / ulp) * ulp
    shrink = (np.sign(x) == np.sign(q)) == against  # the magnitude must round down
    mag = lo + 0.5 * ulp + np.where(shrink, -1.0, 1.0) * ulp / 1024
    return np.sign(x) * mag


def test_cosine_raw_overwrite_near_the_kth_boundary_keeps_the_proof_sound():
    """brute_force_single.h:139-144 overwrites an existing label with the caller's RAW blob, so a cosine index can hold
    non-unit rows.  Rows of norm ~16 are planted right at the k-th boundary of each query (on both sides of it): their
    fp16 error is ~16x the unit-vector bound, so a proof that assumed unit vectors could pass on a wrong answer.  ids and
    score bits must still equal the reference's."""
    _raw_overwrite_near_the_kth_boundary("random")


def test_cosine_raw_overwrite_with_adversarial_rounding_keeps_the_proof_sound():
    """The same planted rows with every component just short of an fp16 rounding midpoint: the rows just inside the k-th
    boundary round outwards and those just outside round inwards, by ~4e-3 each — beyond the unit-vector window
    2 eps = 2.4e-3, so a bound that lost its norm scaling would pass the proof on a wrong answer."""
    _raw_overwrite_near_the_kth_boundary("adversarial")


def _raw_overwrite_near_the_kth_boundary(rounding):
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 128, 32, 10
    rows = ol.synth_rows(ol.F32, 27, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS)(dim)
    g.add_many(rows, label0=1)
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 28, 0, nq, dim)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    _device_batch(vs, torch, g, qn, k)  # shadow built while every row is still a unit vector
    rng = np.random.default_rng(5)
    scale = 16.0
    victim = 100
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        d_k = float(ps[-1])
        for delta in (-3e-4, -2e-5, 2e-5, 3e-4):  # just inside / just outside the current k-th distance
            want = d_k + delta  # 1 - scale * c = want
            c = (1.0 - want) / scale
            q = qn[i].astype(np.float64)
            u = rng.standard_normal(dim)
            u -= u.dot(q) * q
            u /= np.linalg.norm(u)
            blob = scale * (c * q + np.sqrt(max(0.0, 1.0 - c * c)) * u)
            if rounding == "adversarial":
                blob = _snap_against(blob, q, against=delta < 0)
                p_ = int(np.argmax(np.abs(q)))  # one component (left off the grid) puts the exact distance back at `want`
                blob[p_] += ((1.0 - want) - blob @ q) / q[p_]
            blob = blob.astype(np.float32)
            victim += 1
            assert g.add(blob, victim) == 0  # label exists: in-place overwrite with the raw blob
            p.add(blob, victim)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    planted = 0
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        planted += int(((pi > 100) & (pi <= victim)).sum())
        assert labels[i].tolist() == pi.tolist(), (i, flags[i], labels[i], pi)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    assert planted >= nq, "the planted rows did not reach the top-k: the test is not exercising the boundary"
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and (hl.astype(np.int64) == labels).all()
    vs.lib().VecSimB200_SetCoarseMode(-1)


def test_coarse_path_falls_back_when_the_margin_is_too_small():
    """Many near-duplicates of the query direction: the 24th-best approximate candidate of a row range is
    within the coarse error bound of the true k-th distance, so the proof must fail and the exact scan answers."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    rng = np.random.default_rng(9)
    n, dim, nq, k = 70_000, 64, 16, 10
    base = rng.uniform(-1, 1, dim).astype(np.float32)
    rows = (base[None, :] + 1e-4 * rng.standard_normal((n, dim))).astype(np.float32)  # all rows almost identical
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
    g.add_many(rows, label0=1)
    p.add_many(rows, 1)
    qs = (base[None, :] + 1e-4 * rng.standard_normal((nq, dim))).astype(np.float32)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None and flags.sum() == 0  # nothing can be proven on this corpus
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
        kth = ps[-1]
        assert {l for l, s in zip(labels[i].tolist(), scores[i].tolist()) if s < kth} == {l for l, s in zip(pi.tolist(), ps.tolist()) if s < kth}
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.parametrize("csz,tier", [(40, 1), (120, 2)])
def test_clustered_corpus_stays_on_the_tensor_core_tiers(csz, tier):
    """Clusters of near-duplicates stored contiguously (one 128-row tile = one candidate list of the coarse kernel).
    Round 1 kept the 24 best rows per list: with 40 near-duplicates the 24th-best is within the error bound of the k-th
    distance, the proof failed and the query paid the 100x slower exact scan.  Now the first tier keeps EVERY row below a
    bound taken from a sample pass, so 40 near-duplicates are simply all kept (tier 1); 120 of them overflow the 96-slot
    list and the second tier (adaptive lists of 128, only for the open queries) proves the answer (tier 2)."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    rng = np.random.default_rng(11)
    n, dim, nq, k = 70_000, 128, 48, 10
    rows = ol.synth_rows(ol.F32, 31, 0, n, dim)
    centers = []
    for c in range(nq):
        start = (8 + 11 * c) * 128 + 4  # every cluster inside one 128-row tile, i.e. one candidate list of the coarse kernel
        center = rng.uniform(-1, 1, dim).astype(np.float32)
        rows[start:start + csz] = center[None, :] + 2e-3 * rng.standard_normal((csz, dim)).astype(np.float32)
        centers.append(center)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = _checker(ol.COS)(dim)
    g.add_many(rows, label0=1)
    p.add_many(rows, 1)
    qs = np.stack([c + 2e-3 * rng.standard_normal(dim).astype(np.float32) for c in centers]).astype(np.float32)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None
    assert (flags == tier).sum() >= nq * 0.9, f"tiers: {np.bincount(flags, minlength=3).tolist()} (exact, tier 1, tier 2)"
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist(), (i, flags[i], labels[i], pi)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.parametrize("fixed", ["0", "1"])
def test_single_pass_adaptive_lists_remain_available(fixed, monkeypatch):
    """VECSIM_B200_FIXED=0 keeps round 1's single pass with adaptive lists (read once per process: checked in a subprocess)."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (
        "import sys, os\n"
        f"sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, 'tests'))\n"
        "import numpy as np, oracle_lib as ol\n"
        "from redisearch_b200 import vecsim as vs\n"
        "n, dim, nq, k = 70000, 128, 40, 10\n"
        "rows = ol.synth_rows(ol.F32, 42, 0, n, dim)\n"
        "g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)\n"
        "p = ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)\n"
        "g.add_many(rows, label0=1); p.add_many(rows, 1)\n"
        "qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)\n"
        "labels, scores, rc = g.topk_batch(qs, k)\n"
        "assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 1\n"
        "for i in range(nq):\n"
        "    pi, ps = p.topk(qs[i], k)\n"
        "    assert labels[i].astype(np.int64).tolist() == pi.tolist()\n"
        "    assert scores[i].astype(np.float32).tobytes() == ps.astype(np.float32).tobytes()\n"
        "print('VARIANT-OK')\n"
    )
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=dict(os.environ, VECSIM_B200_FIXED=fixed))
    assert r.returncode == 0 and "VARIANT-OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.parametrize("n,dim,nq,k", [(70_000, 128, 40, 32), (66_000, 768, 64, 100), (131_072, 96, 17, 128)])
def test_fp32_coarse_route_serves_k_up_to_128(n, dim, nq, k):
    """k > 16 on the fp32 route: lists of 128 per row range from the start (round 1 sent these batches to the 414 ms
    CUDA-core scan); ids and score bits equal to the oracle."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qn = qs.copy()
    for i in range(nq):
        ol.port().orc_normalize(ol._p(qn[i]), dim, ol.F32)
    labels, scores, flags = _device_batch(vs, torch, g, qn, k)
    assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    assert (flags != 0).sum() >= nq * 0.9
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist(), (i, flags[i])
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.parametrize("vtype,metric,n,dim,nq,k", [(ol.F16, ol.IP, 70_000, 128, 40, 10), (ol.BF16, ol.COS, 66_000, 768, 130, 100),
                                                     (ol.F16, ol.COS, 140_000, 96, 300, 32), (ol.BF16, ol.IP, 70_000, 256, 17, 128)])
def test_16bit_corpora_take_the_tensor_core_route(vtype, metric, n, dim, nq, k):
    """fp16 / bf16 corpora (BASELINE configs[2] shape): the batched query is one wgmma GEMM with fused top-k, its
    fp32-accumulated products are the distances.  Bar (BASELINE north_star): scores within 1e-2, ids identical modulo
    candidates within that tolerance of the k-th; observed agreement with the fp32-accumulate reference tier ~1e-6."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    vt = {ol.F16: vs.VecSimType_FLOAT16, ol.BF16: vs.VecSimType_BFLOAT16}[vtype]
    mt = {ol.IP: vs.VecSimMetric_IP, ol.COS: vs.VecSimMetric_Cosine}[metric]
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    g = vs.VecSimIndex(vt, dim, mt)
    p = ol.PortIndex(vtype, dim, metric, tier=ol.TIER_AVX512)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    labels, scores, rc = g.topk_batch(qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 2
    worst = 0.0
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert len(pi) == k
        for a, e in zip(scores[i], ps):
            assert abs(a - e) <= 1e-2 * max(abs(e), 1.0) + 1e-6
            worst = max(worst, abs(a - e) / max(abs(e), 1.0))
        kth = ps[-1]
        slack = 1e-2 * max(abs(kth), 1.0) + 1e-6
        sure = {int(l) for l, s in zip(pi.tolist(), ps.tolist()) if s < kth - slack}
        assert sure <= {int(x) for x in labels[i].tolist()}
        # in practice the two agree far better than the bar: identical ids wherever the oracle has no near-tie
        gaps = np.diff(ps)
        if (gaps > 1e-4).all():
            assert labels[i].astype(np.int64).tolist() == pi.tolist()
    assert worst < 1e-4, worst
    # the exact CUDA-core scan gives the same answer within the same bar
    vs.lib().VecSimB200_SetCoarseMode(0)
    l2, s2, rc = g.topk_batch(qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 0
    assert np.abs(s2 - scores).max() <= 1e-4
    vs.lib().VecSimB200_SetCoarseMode(-1)


def test_16bit_fixed_bound_pass_and_its_second_tier():
    """fp16 corpora: the batched scan is a sample pass + a fixed-bound main pass (every row with distance <= the bound is kept in
    lists of 256 per row range, no compaction).  Uniform data stays on that tier (flag 1); 300 near-duplicates of the query
    direction packed into ONE row range overflow its list and the adaptive kernel answers (flag 2).  Either way the distances
    are within the 1e-2 bar of the reference tier and every id whose distance is clearly below the k-th is present."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 140_000, 96, 32, 10
    rng = np.random.default_rng(3)
    rows32 = ol.synth_rows(ol.F32, 42, 0, n, dim)
    base = rng.uniform(-1, 1, dim).astype(np.float32)
    # nq <= 64: one query group, one row range per SM (plan_coarse: grid_x = min(tiles, SMs)); tiles t, t + gx, t + 2 gx share a range
    gx = torch.cuda.get_device_properties(0).multi_processor_count
    for j, t in enumerate((5, 5 + gx, 5 + 2 * gx)):
        rows32[t * 128:t * 128 + 100] = 3.0 * base[None, :] + 1e-2 * rng.standard_normal((100, dim)).astype(np.float32)
    rows = rows32.astype(np.float16).view(np.uint16)  # round-to-nearest-even, like the reference's float16.h conversion
    g = vs.VecSimIndex(vs.VecSimType_FLOAT16, dim, vs.VecSimMetric_IP)
    p = ol.PortIndex(ol.F16, dim, ol.IP, tier=ol.TIER_AVX512)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    # uniform queries, flipped away from the planted direction where needed: a query that happens to point along `base` sees all
    # 300 planted rows (3x the norm of the rest) at the top, which rightly overflows the range's list like the cluster queries do
    uniform_q32 = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    uniform_q32[(uniform_q32 @ base) > 0] *= -1.0
    uniform_q = uniform_q32.astype(np.float16).view(np.uint16)
    cluster_q = (base[None, :] + 1e-2 * rng.standard_normal((nq, dim))).astype(np.float16).view(np.uint16)
    for qs, want in ((uniform_q, 1), (cluster_q, 2)):
        qd = torch.from_numpy(qs.view(np.int16)).cuda()
        out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
        torch.cuda.synchronize()
        assert vs.lib().VecSimB200_LastBatchPath(g.h) == 2
        flags = np.zeros(nq, dtype=np.uint32)
        assert vs.lib().VecSimB200_LastCoarseFlags(g.h, flags.ctypes.data, nq) == 0
        assert (flags == want).sum() >= nq * 0.9, (want, np.bincount(flags, minlength=3).tolist())
        labels, scores = out_l.cpu().numpy(), out_s.cpu().numpy()
        for i in range(nq):
            pi, ps = p.topk(qs[i], k)
            assert np.abs(scores[i] - ps.astype(np.float32)).max() <= 1e-2 * max(1.0, float(np.abs(ps).max()))
            kth = float(ps[-1])
            safe = {int(l) for l, s_ in zip(pi.tolist(), ps.tolist()) if s_ < kth - 1e-2 * max(1.0, abs(kth))}
            assert safe <= set(labels[i].tolist()), (want, i)
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.parametrize("vtype,metric,n,dim,nq,k", [(ol.I8, ol.COS, 70_000, 128, 40, 10), (ol.I8, ol.IP, 66_000, 768, 130, 100),
                                                     (ol.U8, ol.COS, 140_000, 96, 300, 32), (ol.U8, ol.IP, 70_000, 256, 17, 128),
                                                     (ol.I8, ol.COS, 66_000, 1024, 64, 10)])
def test_8bit_corpora_take_the_integer_tensor_core_route_bit_exact(vtype, metric, n, dim, nq, k):
    """int8 / uint8 corpora: s8 / u8 wgmma dot products are exact int32 sums and the epilogue applies the reference's
    float expression (IP.cpp:248-285), so ids AND score bits must equal the oracle's — including tie order by id."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    vt = {ol.I8: vs.VecSimType_INT8, ol.U8: vs.VecSimType_UINT8}[vtype]
    mt = {ol.IP: vs.VecSimMetric_IP, ol.COS: vs.VecSimMetric_Cosine}[metric]
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    rows[5000:5040] = rows[4000:4040]  # exact duplicates: ties that must resolve to the lower id
    g = vs.VecSimIndex(vt, dim, mt)
    p = ol.PortIndex(vtype, dim, metric, tier=ol.TIER_AVX512)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[1] = rows[4003]  # a query whose best hits are a tied pair
    labels, scores, rc = g.topk_batch(qs, k)
    assert rc == 0 and vs.lib().VecSimB200_LastBatchPath(g.h) == 2
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].astype(np.int64).tolist() == pi.tolist(), (i, labels[i][:12], pi[:12])
        assert scores[i].astype(np.float32).tobytes() == ps.astype(np.float32).tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)


def test_single_queries_ride_the_shadow_once_a_batch_built_it():
    """VecSimIndex_TopKQuery (one query) takes the coarse route only when an up-to-date fp16 shadow already exists;
    the answer is the exact scan's either way, and a mutation sends single queries back to the exact scan until the
    next batch refreshes the shadow."""
    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, k = 70_000, 128, 10
    rows = ol.synth_rows(ol.F32, 42, 0, n + 10, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    p = ol.PortIndex(ol.F32, dim, ol.COS, tier=ol.TIER_AVX512)
    g.add_many(rows[:n], label0=1)
    p.add_many(rows[:n], 1)
    qs = ol.synth_rows(ol.F32, 43, 0, 20, dim)

    def check_single(expect_path):
        for q in qs[:6]:
            gi, gs, code = g.topk(q, k)
            pi, ps = p.topk(q, k)
            assert code == 0 and gi.tolist() == pi.tolist()
            assert gs.astype(np.float32).tobytes() == ps.astype(np.float32).tobytes()
            assert vs.lib().VecSimB200_LastBatchPath(g.h) == expect_path

    check_single(0)                     # no shadow yet: exact scan
    g.topk_batch(qs, k)                 # a batch builds it
    assert vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    check_single(1)
    g.add(rows[n], n + 1)               # stale shadow: single queries do not pay for the refresh
    p.add(rows[n], n + 1)
    check_single(0)
    g.topk_batch(qs, k)
    check_single(1)
    vs.lib().VecSimB200_SetCoarseMode(-1)


@pytest.mark.parametrize("metric,n,dim,nq,k", [(ol.L2, 70_000, 128, 40, 10), (ol.IP, 66_000, 768, 130, 10), (ol.L2, 140_000, 96, 300, 16),
                                               (ol.L2, 66_000, 768, 64, 10)])
def test_fp32_l2_and_raw_ip_batches_take_the_coarse_route_exactly(metric, n, dim, nq, k):
    """fp32 L2 / raw inner product: same coarse-then-exact pipeline, the GEMM runs on the fp16 shadow of the raw rows, squared
    L2 is assembled from the dot product and the squared norms, and the proof's error bound scales with the row / query
    norms.  ids and score bits must equal the oracle's exact scan."""
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    mt = {ol.L2: vs.VecSimMetric_L2, ol.IP: vs.VecSimMetric_IP}[metric]
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, mt)
    p = ol.PortIndex(ol.F32, dim, metric, tier=ol.TIER_AVX512)
    assert g.add_many(rows, label0=1) == n
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    labels, scores, flags = _device_batch(vs, torch, g, qs, k)
    assert vs.lib().VecSimB200_LastBatchPath(g.h) == 1 and flags is not None
    assert (flags != 0).sum() >= nq * 0.9, f"only {int(flags.sum())}/{nq} queries were verified by the coarse path"
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist(), (i, flags[i], labels[i], pi)
        assert scores[i].tobytes() == ps.astype(np.float32).tobytes()
    # a single query rides the same shadow
    gi, gs, code = g.topk(qs[0], k)
    pi, ps = p.topk(qs[0], k)
    assert code == 0 and gi.tolist() == pi.tolist() and gs.astype(np.float32).tobytes() == ps.astype(np.float32).tobytes()
    assert vs.lib().VecSimB200_LastBatchPath(g.h) == 1
    vs.lib().VecSimB200_SetCoarseMode(-1)


def test_values_outside_the_fp16_range_keep_l2_batches_on_the_exact_scan():
    import torch

    from redisearch_b200 import vecsim as vs

    vs.lib().VecSimB200_SetCoarseMode(1)
    n, dim, nq, k = 70_000, 64, 32, 10
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    rows[123, 5] = 1.0e5  # does not fit an IEEE half
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_L2)
    p = ol.PortIndex(ol.F32, dim, ol.L2, tier=ol.TIER_AVX512)
    g.add_many(rows, label0=1)
    p.add_many(rows, 1)
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    labels, scores, flags = _device_batch(vs, torch, g, qs, k)
    assert vs.lib().VecSimB200_LastBatchPath(g.h) == 0 and flags is None
    for i in range(nq):
        pi, ps = p.topk(qs[i], k)
        assert labels[i].tolist() == pi.tolist() and scores[i].tobytes() == ps.astype(np.float32).tobytes()
    vs.lib().VecSimB200_SetCoarseMode(-1)
