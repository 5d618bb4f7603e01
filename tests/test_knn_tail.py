"""The int8 KNN route past its main pass (DESIGN.md §4.2): the sample pass runs on the main pass's 128-query CTAs with slice
minima taken from the accumulator fragment, and the fixed-bound main pass publishes a count per (query, row range) in place of
padding its lists, which refine_kernel gathers into shared memory (or, above its cap, reads from global memory).

Batches on that route must answer exactly as the exact scan of the same index, label and score bits, and the first tier must
prove every query, across dimensions (256, 768, 1024), batch sizes that split into CTAs in every way (16, 129, 256, 1000) and k
(1, 10, 128), over a corpus whose last row tile is partly filled.  A query whose lists hold more live entries than the shared
memory takes is answered from the lists in global memory and still proven.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol

_N = 65_536 + 77  # the last row tile holds 77 rows
_indexes = {}


def _index(vs, dim):
    if dim not in _indexes:
        _indexes.clear()  # one corpus at a time on the device
        g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
        assert g.add_many(ol.synth_rows(ol.F32, 52, 0, _N, dim), label0=1) == _N
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


_CASES = [(dim, nq, k) for dim in (256, 768, 1024) for nq in (16, 129, 256, 1000) for k in (1, 10, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nq,k", _CASES)
def test_int8_route_is_exact_and_proven_by_tier_1(dim, nq, k):
    import torch

    from redisearch_b200 import vecsim as vs

    g = _index(vs, dim)
    flags = _check_against_exact(vs, torch, g, ol.synth_rows(ol.F32, 53, 0, nq, dim), k)
    assert (flags == 1).all(), np.bincount(flags)


@pytest.mark.gpu
def test_live_entries_past_the_shared_memory_cap_are_read_from_global_memory():
    """Query 7 lies near one centre c.  128 rows sit at cosine 0.9 from c and 10,000 at cosine 0.75, scattered over the
    corpus.  The sample pass's bound for query 7 sits near the crowd (it visits a quarter of the tiles, which hold about 32 of
    the 128 near rows), so the main pass keeps the whole crowd: about 10,100 live entries, above refine_kernel's 8,192 in
    shared memory, and about 150 per list of 256, so no list overflows.  The rescoring then reads the lists in global memory;
    its survivors are the 128 near rows, far below the crowd, and the first tier proves the answer.  The other queries are
    random."""
    import torch

    from redisearch_b200 import vecsim as vs

    rng = np.random.default_rng(31)
    dim, nq, k = 256, 256, 128
    n_bg, n_crowd, n_near = 140_000, 10_000, 128
    c = rng.standard_normal(dim)
    c /= np.linalg.norm(c)

    def around(n, cos_t):  # unit rows at cosine cos_t from c, in random directions orthogonal to it
        u = rng.standard_normal((n, dim))
        u -= np.outer(u @ c, c)
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        return (cos_t * c + np.sqrt(1 - cos_t * cos_t) * u).astype(np.float32)

    rows = np.concatenate([ol.synth_rows(ol.F32, 42, 0, n_bg, dim), around(n_crowd, 0.75), around(n_near, 0.9)])
    rows = np.ascontiguousarray(rows[rng.permutation(rows.shape[0])])
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    qs[7] = c.astype(np.float32)
    q7 = _normalized(qs[7:8])[0].astype(np.float64)
    cos = (rows.astype(np.float64) @ q7) / np.linalg.norm(rows.astype(np.float64), axis=1)
    assert (cos > 0.7).sum() > 8192 + 1000 and (cos > 0.85).sum() == n_near
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, vs.VecSimMetric_Cosine)
    assert g.add_many(rows, label0=1) == rows.shape[0]
    flags = _check_against_exact(vs, torch, g, qs, k)
    assert flags[7] == 1, flags[7]
    assert (flags != 0).sum() >= nq * 0.9, np.bincount(flags)
