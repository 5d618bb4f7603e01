"""The int8 copy of unit fp32 rows (cosine batches with k <= 128, DESIGN.md §4.2): the approximate pass runs on int8 operands with
one scale per 128-row tile and a per-query error bound; rescoring stays in fp32, so labels and score bits must equal the exact
scan's whatever tier answers.

The first test is CPU-only: a numpy restatement of the quantization and of the bound of quantize_queries_kernel, checked in
fp64 on rows and queries built to make the rounding errors add up.  The others run on the GPU against the exact scan of the
same index (coarse mode 0), which the rest of the suite holds to the reference bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol


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


def test_int8_bound_covers_worst_case_rounding():
    """|approx - exact| <= eps_q in fp64 for rows and queries at rounding midpoints with aligned signs, and the distance the kernel
    computes in fp32, 1 - fl(fl(s_q s_t) acc), stays within eps_q of the fp64 distance."""
    rng = np.random.default_rng(7)
    worst = 0.0
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
                worst = max(worst, abs(approx64 - exact) / eps)
    assert worst > 0.05, worst  # the construction does push the error towards the bound


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
