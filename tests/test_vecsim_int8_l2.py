"""int8 / uint8 L2 KNN batches on the integer tensor cores (coarse_wgmma_kernel kOp 4, DESIGN.md §3 and §4).

The reference computes float(sum of (a_i - q_i)^2) over int32 (L2.cpp:148-174).  s8 / u8 wgmma gives a.q exactly, the index
keeps the exact int32 |row|^2 of every row and the batch computes |q|^2, so __int2float_rn(|a|^2 + |q|^2 - 2 a.q) is that
float bit for bit.  Selection keys are built on the float, so integer distances above 2^24 that round to the same float are
ties and resolve by row id, as in the reference's heap.

GPU: every answer must equal the reference's own scan (Ref_ScanTopKChunk, when oracle/_ref is built; else the C restatement)
and ol.PortIndex at the AVX-512 tier in ids and float32 score bits, and every eligible batch reports LastBatchPath == 2.
CPU: the tie builder has its power, and the int32 range argument holds at the widest dim the route takes.
"""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as ol

_VT = {ol.I8: 4, ol.U8: 5}  # VecSimType_INT8 / UINT8
_L2 = 0                     # VecSimMetric_L2
MAX_DIM = 2048              # widest 8-bit row the main pass keeps two ring stages for (coarse_tc.cu wgmma_fits_bytes)
SIZE_MAX = np.uint64(0xFFFFFFFFFFFFFFFF)


def _vs():
    from redisearch_b200 import vecsim as vs

    return vs


@pytest.fixture
def mode1():
    vs = _vs()
    vs.lib().VecSimB200_SetCoarseMode(1)
    yield vs
    vs.lib().VecSimB200_SetCoarseMode(-1)


# ------------------------------------------------------------------------------------------------------------------
# builders (CPU)
# ------------------------------------------------------------------------------------------------------------------
def _as_type(s, vtype):
    """Offsets s in [0, 255] from the type's minimum -> stored values (int8: s - 128, uint8: s)."""
    s = np.asarray(s, dtype=np.int64)
    return (s - 128).astype(np.int8) if vtype == ol.I8 else s.astype(np.uint8)


def _four_squares(t, rng):
    """a, b, c, d in [0, 255] with a^2 + b^2 + c^2 + d^2 == t (t <= 4 * 255^2); random start, then a scan."""
    for a in list(rng.permutation(256)):
        ra = t - a * a
        if ra < 0:
            continue
        for b in range(256):
            rb = ra - b * b
            if rb < 0:
                break
            for c in range(256):
                rc = rb - c * c
                if rc < 0:
                    break
                d = int(round(rc ** 0.5))
                if d * d == rc and d <= 255:
                    return [int(a), b, c, d]
    raise AssertionError(f"no four squares for {t}")


def tie_rows(vtype, dim, n_pairs, seed=0):
    """A query at the type's minimum in every component and pairs of rows (A, B) far from it whose integer squared distances
    are D + 1 (A) and D - 1 (B) for a D where the float spacing is >= 4, so both round to the same float D.  A goes before B in
    the corpus: the lower id holds the LARGER integer.  A selection on the integer would rank B first; the reference ranks A
    first (equal floats, lower id).  Every other component of the pair is at the type's maximum, 8 components are free, and the
    pairs are nearer the query than the filler rows of filler_rows().  Returns (query, [(row_a, row_b, D)])."""
    rng = np.random.default_rng(seed)
    q = _as_type(np.zeros(dim), vtype)
    base = (dim - 8) * 255 * 255
    pairs = []
    for j in range(n_pairs):
        D = ((base + 4 * 100 * 100) // 64 + j) * 64  # a multiple of the float spacing (<= 16 up to dim 2048)
        rows = []
        for t in (D + 1, D - 1):
            rest = t - base
            s = np.full(dim, 255, dtype=np.int64)
            s[dim - 8:dim - 4] = _four_squares(rest // 2, rng)
            s[dim - 4:] = _four_squares(rest - rest // 2, rng)
            perm = rng.permutation(dim)  # spread the free components over the row
            rows.append(_as_type(s[perm], vtype))
        pairs.append((rows[0], rows[1], D))
    return q, pairs


def filler_rows(vtype, dim, n, seed=1):
    """Rows at the type's maximum except 4 random components in [200, 255] (offsets): their distance to the minimum query is
    at least dim * 65025 - 4 * (65025 - 40000), farther than every tie pair (which sits 8 * 65025 - ~40000 below the maximum)."""
    rng = np.random.default_rng(seed)
    s = np.full((n, dim), 255, dtype=np.int64)
    cols = rng.integers(0, dim, (n, 4))
    s[np.arange(n)[:, None], cols] = rng.integers(200, 256, (n, 4))
    return _as_type(s, vtype)


def _l2_int(a, b):
    d = a.astype(np.int64) - b.astype(np.int64)
    return int((d * d).sum())


# ------------------------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("dim", [1024, MAX_DIM])
def test_tie_builder_has_its_power(vtype, dim):
    q, pairs = tie_rows(vtype, dim, 3)
    filler = filler_rows(vtype, dim, 64)
    worst_pair = 0
    for a, b, D in pairs:
        da, db = _l2_int(a, q), _l2_int(b, q)
        assert da == D + 1 and db == D - 1 and da > db  # the integers differ, the lower id (a) holds the larger one
        assert np.float32(da) == np.float32(db) == np.float32(D) and D > 2 ** 24  # ... and the floats are equal
        worst_pair = max(worst_pair, da)
    assert min(_l2_int(r, q) for r in filler) > worst_pair  # the pairs are the nearest rows


@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_int32_range_at_the_widest_dim(vtype):
    """|a|^2 + |q|^2 - 2 a.q as the kernel evaluates it ((|a|^2 + |q|^2) - 2 dot, and |a|^2 + |q|^2 - 2 dot in the pre-test) stays
    inside int32 for every pair of rows at dim 2048, and equals the exact sum of squared differences."""
    lo, hi = (-128, 127) if vtype == ol.I8 else (0, 255)
    dim = MAX_DIM
    rng = np.random.default_rng(5)
    cands = [np.full(dim, lo), np.full(dim, hi), np.zeros(dim, dtype=np.int64), rng.integers(lo, hi + 1, dim), rng.integers(lo, hi + 1, dim)]
    alt = np.full(dim, lo)
    alt[::2] = hi
    cands.append(alt)
    bound = 0
    for a in cands:
        for q in cands:
            a64, q64 = a.astype(np.int64), q.astype(np.int64)
            na, nq, dot = int(a64 @ a64), int(q64 @ q64), int(a64 @ q64)
            for v in (na, nq, dot, 2 * dot, na + nq, na + nq - 2 * dot, na - 2 * dot):
                assert -2 ** 31 <= v < 2 ** 31
                bound = max(bound, abs(v))
            assert na + nq - 2 * dot == _l2_int(a, q)
            # the same in wrapping int32 arithmetic, then one rounding to float: the reference's float
            i32 = (np.int32(na) + np.int32(nq)) - np.int32(2) * np.int32(dot)
            assert np.float32(i32) == np.float32(_l2_int(a, q))
    # worst case over all inputs: 2 * 255^2 * dim for uint8 (|a|^2 + |q|^2 with a = q = 255), half that for int8 (2 * 128^2 * dim)
    assert bound <= 2 * 255 * 255 * dim < 2 ** 31


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _index(vtype, dim, rows, multi=False, labels=None):
    vs = _vs()
    g = vs.VecSimIndex(_VT[vtype], dim, _L2, multi=multi)
    p = ol.PortIndex(vtype, dim, ol.L2, multi=multi, tier=ol.TIER_AVX512)
    if labels is None:
        assert g.add_many(rows, label0=1) == len(rows)
        p.add_many(rows, 1)
    else:
        assert g.add_many(rows, labels=labels) == len(rows)
        for r, lab in zip(rows, labels.tolist()):
            p.add(r, lab)
    return g, p


def _stream_oracle(vtype, dim, rows, qs, k):
    """The reference's own distance kernel + heap over rows labelled 1.. (Ref_ScanTopKChunk), or the C restatement."""
    s = ol.StreamingTopK(vtype, ol.L2, dim, qs, k, os.cpu_count() or 1)
    s.feed(rows, 1)
    return s


def _check(g, p, qs, k, labels, scores, stream=None, port_queries=None):
    """ids and float32 score bits against the streaming oracle (every query) and PortIndex (the listed queries, default all)."""
    nq = qs.shape[0]
    for i in range(nq):
        h = int((labels[i] != SIZE_MAX).sum())
        gi, gs = labels[i, :h].astype(np.int64), scores[i, :h].astype(np.float32)
        if stream is not None:
            si, ss = stream.result(i)
            assert gi.tolist() == si.tolist(), (i, gi[:8].tolist(), si[:8].tolist())
            assert gs.tobytes() == ss.astype(np.float32).tobytes(), i
        if port_queries is None or i in port_queries:
            pi, ps = p.topk(qs[i], k)
            assert gi.tolist() == pi.tolist(), (i, gi[:8].tolist(), pi[:8].tolist())
            assert gs.tobytes() == ps.astype(np.float32).tobytes(), i


def _path(g):
    return _vs().lib().VecSimB200_LastBatchPath(g.h)


def _device_batch(g, qs, k):
    import torch

    vs = _vs()
    nq, dim = qs.shape
    pitch = (dim + 15) // 16 * 16  # the device API reads query i at i * round16(stored bytes)
    buf = np.zeros((nq, pitch), dtype=np.uint8)
    buf[:, :dim] = np.ascontiguousarray(qs).view(np.uint8)
    qd = torch.from_numpy(buf).cuda()
    out_l = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    out_s = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp)
    torch.cuda.synchronize()
    assert rc == 0
    return out_l.cpu().numpy(), out_s.cpu().numpy()


_BATCHES = [(16, 1), (40, 10), (256, 100), (17, 128)]


# ------------------------------------------------------------------------------------------------------------------
# GPU: parity matrix
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("dim", [32, 128, 768, 1024, MAX_DIM])
@pytest.mark.parametrize("n", [66_000, 140_000])
def test_matrix_is_bit_exact(mode1, vtype, dim, n):
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    rows[5000:5040] = rows[4000:4040]  # exact duplicates: the lower id wins
    rows[n - 300:n - 260] = rows[4000:4040]  # ... also across row ranges
    g, p = _index(vtype, dim, rows)
    qs_all = ol.synth_rows(vtype, 43, 0, 256, dim)
    qs_all[1] = rows[4003]  # a query equal to a row: distance 0, three tied rows
    qs_all[2] = rows[n - 1]  # ... and to the last row
    for nq, k in _BATCHES:
        qs = np.ascontiguousarray(qs_all[:nq])
        labels, scores, rc = g.topk_batch(qs, k)
        assert rc == 0 and _path(g) == 2, (nq, k)
        assert labels[1, 0] == 4004 and scores[1, 0] == 0.0
        _check(g, p, qs, k, labels, scores, _stream_oracle(vtype, dim, rows, qs, k), port_queries={0, 1, 2, nq - 1})


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_extreme_values_at_the_widest_dim(mode1, vtype):
    """int8 -128 against 127 and uint8 0 against 255 in every component: the largest distance there is, 65025 * 2048."""
    dim, n, nq, k = MAX_DIM, 66_000, 32, 100
    lo, hi = (-128, 127) if vtype == ol.I8 else (0, 255)
    rows = np.full((n, dim), hi, dtype=ol.NP_DTYPE[vtype])
    rows[1000:1020] = lo
    rows[30_000:30_030] = ol.synth_rows(vtype, 42, 0, 30, dim)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[: nq // 2] = lo
    qs[nq // 2:] = hi
    qs[3] = rows[30_007]  # a random row among the extremes
    g, p = _index(vtype, dim, rows)
    labels, scores, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 2
    assert scores[0, 0] == 0.0 and scores[nq - 1, 0] == 0.0  # the query's own extreme rows
    # a query at the minimum sees 20 rows at 0, 30 random rows and then rows at the maximum distance, 65025 * dim, tied by id
    far = np.float32(65025 * dim)
    assert (scores[0] == far).sum() == k - 50 and (labels[0, 50:] == np.arange(1, k - 49, dtype=np.uint64)).all()
    _check(g, p, qs, k, labels, scores, _stream_oracle(vtype, dim, rows, qs, k), port_queries={0, 3, nq - 1})


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_float_rounding_ties_resolve_by_row_id(mode1, vtype):
    """Rows whose integer distances differ (D + 1 and D - 1) but round to the same float: the lower id, which holds the LARGER
    integer, must come first, as in the reference.  Pairs are spread over the corpus (different row ranges of the main pass)."""
    dim, n, k = 1024, 66_000, 20
    q, pairs = tie_rows(vtype, dim, 8)
    rows = filler_rows(vtype, dim, n)
    where = [100, 7_000, 20_000, 33_333, 47_000, 60_000, 64_000, 65_800]
    for (a, b, _), at in zip(pairs, where):
        rows[at], rows[at + 1 + (at % 97)] = a, b
    qs = np.repeat(q[None, :], 16, axis=0)
    g, p = _index(vtype, dim, rows)
    for kk in (1, k):
        labels, scores, rc = g.topk_batch(qs, kk)
        assert rc == 0 and _path(g) == 2
        _check(g, p, qs, kk, labels, scores, _stream_oracle(vtype, dim, rows, qs, kk), port_queries={0})
        # the first pair: A (row where[0], label where[0] + 1) before B, at the same float score
        assert labels[0, 0] == where[0] + 1
        if kk > 1:
            assert labels[0, 1] == where[0] + 2 + where[0] % 97 and scores[0, 0] == scores[0, 1] == np.float32(pairs[0][2])


# ------------------------------------------------------------------------------------------------------------------
# GPU: batches that leave the route
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("case", ["dim", "nq", "rows", "mode0"])
def test_batches_off_the_route_answer_the_same(mode1, vtype, case):
    dim = MAX_DIM + 16 if case == "dim" else 128
    n = 65_535 if case == "rows" else 66_000
    nq, k = (15 if case == "nq" else 32), 10
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    rows[5000:5040] = rows[4000:4040]
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[1] = rows[4003]
    g, p = _index(vtype, dim, rows)
    if case == "mode0":
        mode1.lib().VecSimB200_SetCoarseMode(0)
    labels, scores, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 0
    _check(g, p, qs, k, labels, scores, _stream_oracle(vtype, dim, rows, qs, k), port_queries={0, 1})
    if case == "mode0":  # the same batch on the route gives the same answer
        mode1.lib().VecSimB200_SetCoarseMode(1)
        l2, s2, rc = g.topk_batch(qs, k)
        assert rc == 0 and _path(g) == 2 and (l2 == labels).all() and s2.tobytes() == scores.tobytes()


# ------------------------------------------------------------------------------------------------------------------
# GPU: mutations between batches keep the |row|^2 table right
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_mutations_between_batches(mode1, vtype):
    """Each step changes rows so that a stale |row|^2 would change the answer: the changed row becomes a copy of a query (distance
    0 only with its new norm; with the old one its score would be |old|^2 - |q|^2), and every step is followed by a batch that
    must equal the reference index that took the same mutations."""
    import torch

    vs = mode1
    dim, n, nq, k = 128, 70_000, 32, 10
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    lo = -128 if vtype == ol.I8 else 0
    g, p = _index(vtype, dim, rows)
    next_label = [n + 1]

    def batch(tag, expect_first=None):
        labels, scores, rc = g.topk_batch(qs, k)
        assert rc == 0 and _path(g) == 2, tag
        _check(g, p, qs, k, labels, scores)
        for qi, lab in (expect_first or {}).items():
            assert labels[qi, 0] == lab and scores[qi, 0] == 0.0, (tag, qi, labels[qi, :3])
        dl, ds = _device_batch(g, qs, k)
        assert (dl.astype(np.uint64) == labels).all() and ds.tobytes() == scores.astype(np.float32).tobytes(), tag

    def both(fn):
        fn(g)
        fn(p)

    batch("fresh")
    # 1. in-place overwrite of a resident row (its norm moves from a random row's to the query's)
    both(lambda x: x.add(qs[0], 777))
    batch("overwrite resident", {0: 777})
    # 2. in-place overwrite of a staged row: append, then overwrite before the next batch
    staged = next_label[0]
    next_label[0] += 1
    both(lambda x: x.add(np.full(dim, lo, dtype=rows.dtype), staged))
    both(lambda x: x.add(qs[1], staged))
    batch("overwrite staged", {1: staged})
    # 3. swap-delete: the last row (a copy of query 2) moves into the hole of label 1000
    last = next_label[0]
    next_label[0] += 1
    both(lambda x: x.add(qs[2], last))
    batch("append")
    both(lambda x: x.delete(1000))
    batch("swap-delete", {2: last})
    # 4. delete the last row (no swap: the staged row of step 2), append a different row that reuses its id
    both(lambda x: x.delete(staged))
    reuse = next_label[0]
    next_label[0] += 1
    both(lambda x: x.add(qs[3], reuse))
    batch("delete + reuse", {3: reuse})
    # 5. AddVectorsDevice: rows appended from device memory, one a copy of query 4
    add = np.ascontiguousarray(ol.synth_rows(vtype, 44, 0, 64, dim))
    add[5] = qs[4]
    d_add = torch.from_numpy(add.view(np.uint8).copy()).cuda()
    label0 = next_label[0]
    next_label[0] += 64
    assert vs.lib().VecSimB200_AddVectorsDevice(g.h, d_add.data_ptr(), 64, label0) == 64
    p.add_many(add, label0)
    batch("device add", {4: label0 + 5})
    # 6. growth past the reserved capacity (the table is reallocated and rebuilt): 1.6x the rows, one a copy of query 5
    more = ol.synth_rows(vtype, 45, 0, 42_000, dim)
    more[41_000] = qs[5]
    label0 = next_label[0]
    both(lambda x: x.add_many(more, label0=label0))
    batch("growth", {5: label0 + 41_000})
    # 7. an in-place overwrite that moves a row AWAY from a query: the old best hit of query 0 must leave the answer
    both(lambda x: x.add(np.full(dim, lo, dtype=rows.dtype), 777))
    batch("overwrite away")


# ------------------------------------------------------------------------------------------------------------------
# GPU: device API and multi-value indexes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
def test_device_api_equals_host_api(mode1, vtype):
    dim, n, nq, k = 768, 66_000, 64, 100
    rows = ol.synth_rows(vtype, 42, 0, n, dim)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[1] = rows[123]
    g, p = _index(vtype, dim, rows)
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 2
    dl, ds = _device_batch(g, qs, k)
    assert _path(g) == 2
    assert (dl.astype(np.uint64) == hl).all() and ds.tobytes() == hs.astype(np.float32).tobytes()
    _check(g, p, qs, k, hl, hs, _stream_oracle(vtype, dim, rows, qs, k), port_queries={0, 1})


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [ol.I8, ol.U8])
@pytest.mark.parametrize("layout", ["independent", "chunks"])
def test_multi_value_indexes(mode1, vtype, layout):
    """Multi-value L2 indexes: the row stage rides the 8-bit L2 route (LastBatchPath 2).  Answers equal the per-query TopKQuery on
    the same index and the multi-value reference (test_vecsim_multi_batch._check_host); the device API equals the host API."""
    from test_vecsim_multi_batch import _check_host

    dim, n, nq, k = 128, 70_002, 40, 10
    rng = np.random.default_rng(9)
    if layout == "independent":  # 3 unrelated rows per label, scattered
        rows = ol.synth_rows(vtype, 42, 0, n, dim)
        labels = np.repeat(1 + 3 * np.arange(n // 3, dtype=np.uint64), 3)[rng.permutation(n)]
    else:  # 6 rows per label, each a small perturbation of the label's centre, contiguous
        per = 6
        centres = ol.synth_rows(vtype, 42, 0, n // per, dim).astype(np.int64)
        noise = rng.integers(-2, 3, (n, dim))
        lo, hi = (-128, 127) if vtype == ol.I8 else (0, 255)
        rows = np.clip(np.repeat(centres, per, axis=0) + noise, lo, hi).astype(ol.NP_DTYPE[vtype])
        labels = np.repeat(1 + np.arange(n // per, dtype=np.uint64), per)
    qs = ol.synth_rows(vtype, 43, 0, nq, dim)
    qs[1] = rows[500]
    g, p = _index(vtype, dim, rows, multi=True, labels=labels)
    hl, hs, rc = g.topk_batch(qs, k)
    assert rc == 0 and _path(g) == 2
    _check_host(g, p, qs, k, hl, hs, True, ol.L2)
    dl, ds = _device_batch(g, qs, k)
    h = hl != SIZE_MAX
    assert ((dl >= 0) == h).all() and (dl[h].astype(np.uint64) == hl[h]).all() and ds[h].tobytes() == hs[h].astype(np.float32).tobytes()
