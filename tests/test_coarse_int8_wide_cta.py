"""The fixed-bound pass over the int8 copy holds 128 queries per CTA (DESIGN.md §4.2): two consumer warpgroups of 64 queries each
run their MMAs against every ring stage, and a batch of 256 runs as clusters of two.  Batches on that route must answer exactly as
the exact scan of the same index, label and score bits, for every way a batch splits into CTAs:

- fewer than 64 queries or exactly 64 (16, 64), and a last CTA of 1 (129) or 72 (200) queries: a warpgroup with no live query,
  which still takes part in every stage of the ring;
- 65, 127, 128: the second warpgroup partly or fully live in a single CTA;
- 256 (two CTAs, a cluster of two), 384 (three: no cluster), 1000 (eight, the last one partly live);

at 136 dimensions (one ring stage per tile), 768 (the benchmark's) and 1024 (the widest the route takes, three ring stages).
Clustered rows that overflow the first tier's lists for queries in both halves of a CTA go to the second tier, which proves them.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol

_N = 65_536 + 300  # a partial last tile
_indexes = {}


def _index(vs, dim):
    if dim not in _indexes:
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        assert g.add_many(ol.synth_rows(ol.F32, 42, 0, _N, dim), label0=1) == _N
        _indexes.clear()  # one corpus at a time on the device
        _indexes[dim] = g
    return _indexes[dim]


def _normalized(qs):
    qn = qs.astype(np.float32).copy()
    for i in range(qn.shape[0]):
        ol.port().orc_normalize(ol._p(qn[i]), qn.shape[1], ol.F32)
    return qn


def _device_batch(vs, torch, index, qn, k):
    nq = qn.shape[0]
    qd = torch.from_numpy(np.ascontiguousarray(qn)).cuda()
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert vs.lib().VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)
    return out_l.cpu().numpy(), out_s.cpu().numpy(), (flags if frc == 0 else None)


def _check_against_exact(vs, torch, g, qs, k):
    """The batch on the int8 copy (asserted) against the exact scan of the same index; returns the per-query tiers."""
    qn = _normalized(qs)
    vs.lib().VecSimB200_SetCoarseMode(1)
    try:
        labels, scores, flags = _device_batch(vs, torch, g, qn, k)
        assert flags is not None and vs.lib().VecSimB200_LastBatchPath(g.h) == 1
        assert vs.lib().VecSimB200_LastCoarseShadowBits(g.h) == 8
        vs.lib().VecSimB200_SetCoarseMode(0)
        el, es, _ = _device_batch(vs, torch, g, qn, k)
    finally:
        vs.lib().VecSimB200_SetCoarseMode(-1)
    for i in range(qs.shape[0]):
        assert labels[i].tolist() == el[i].tolist(), (i, flags[i], labels[i], el[i])
        assert scores[i].tobytes() == es[i].tobytes(), (i, flags[i])
    return flags


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nq,k", [(768, 16, 10), (768, 64, 10), (768, 65, 10), (768, 127, 10), (768, 128, 10), (768, 129, 10),
                                      (768, 200, 10), (768, 256, 10), (768, 384, 10), (768, 1000, 10), (768, 256, 128),
                                      (136, 65, 10), (136, 256, 1), (136, 384, 10),
                                      (1024, 129, 10), (1024, 256, 10), (1024, 1000, 10)])
def test_wide_cta_batches_are_exact(dim, nq, k):
    import torch

    from redisearch_b200 import vecsim as vs

    g = _index(vs, dim)
    flags = _check_against_exact(vs, torch, g, ol.synth_rows(ol.F32, 43, 0, nq, dim), k)
    assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags)


@pytest.mark.gpu
def test_overflow_in_both_halves_of_a_cta_is_proven_by_tier_2():
    """Queries 5 and 70 (the two warpgroups of the first CTA) and 130 and 250 (of the second) lie near one centre.  27,000
    contiguous rows sit at cosine distance 0.3 from it, at least three tiles in every row range, so more rows than a list holds
    fall below each of those queries' fixed bound and the first tier overflows.  24 rows much closer to the centre hold the answer,
    clear of the crowd by far more than the error bound, so the second tier's lists of 128 prove it.  The other queries are
    random."""
    import torch

    from redisearch_b200 import vecsim as vs

    rng = np.random.default_rng(21)
    dim, nq, k = 384, 256, 10
    n_bg, n_far, n_near = 70_000, 27_000, 24
    c = rng.standard_normal(dim)
    c /= np.linalg.norm(c)

    def around(n, cos_t):  # unit rows at cosine cos_t from c, in random directions orthogonal to it
        u = rng.standard_normal((n, dim))
        u -= np.outer(u @ c, c)
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        return (cos_t * c + np.sqrt(1 - cos_t * cos_t) * u).astype(np.float32)

    bg = ol.synth_rows(ol.F32, 42, 0, n_bg, dim)
    far, near = around(n_far, 0.7), around(n_near, 0.98)
    rows = np.ascontiguousarray(np.concatenate([bg[:40_000], far[:13_000], near, far[13_000:], bg[40_000:]]))
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == rows.shape[0]
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    crowded = [5, 70, 130, 250]
    qs[crowded] = around(len(crowded), 0.9999)
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert (flags[crowded] == 2).all(), flags[crowded]
    assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags)
