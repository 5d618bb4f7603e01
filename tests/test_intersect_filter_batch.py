"""Filter-mode ANDs over posting lists and pending sets on the device with no host wait: II_IntersectFilterBatchDevice, alone,
composed with itself, and feeding VecSimB200_TopKFilteredBatchDevice.

Every set must hold the docIds II_IntersectEx gives over the same lists plus II_PostingList_FromDevice of each set child, and
numpy's intersect1d / setdiff1d; its num_estimated (DeviceLen[1]) and child order must follow Intersection::new's rule over the
children's settled estimates; every KNN row fed from it must equal VecSimB200_TopKFiltered on the host-built filter, bit for bit.
"""
import ctypes as C
import os
import re
import subprocess
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32_MAX_ID = 2**32 - 2


def _ps():
    from redisearch_b200 import postings as ps

    return ps


# ------------------------------------------------------------------------------------------------
# CPU: the ABI and the refusals (before the library looks for a device)
# ------------------------------------------------------------------------------------------------
def test_symbol_prototype_and_child_layout(tmp_path):
    ps = _ps()
    assert hasattr(ps.lib(), "II_IntersectFilterBatchDevice")
    hdr = open(os.path.join(ROOT, "include", "ii_b200.h")).read()
    assert re.search(r"int\s+II_IntersectFilterBatchDevice\s*\(\s*size_t nq,\s*const II_FilterChild \*const \*children,\s*"
                     r"const size_t \*n_children,\s*void \*stream,\s*II_ResultSet \*\*out,\s*size_t \*built\)\s*;", hdr)
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "%s"\nint main(void) {\n'
                   '  printf("%%zu %%zu %%zu %%zu\\n", sizeof(II_FilterChild), offsetof(II_FilterChild, list),\n'
                   '         offsetof(II_FilterChild, set), offsetof(II_FilterChild, mode));\n  return 0;\n}\n'
                   % os.path.join(ROOT, "include", "ii_b200.h"))
    exe = tmp_path / "probe"
    subprocess.run(["gcc", str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    F = ps.II_FilterChild
    assert got == [C.sizeof(F), F.list.offset, F.set.offset, F.mode.offset]


def _raw_call(queries, nq=None, null=()):
    """II_IntersectFilterBatchDevice over queries[q] = [(list address, set address, mode)]; `null` names arguments passed as NULL"""
    ps = _ps()
    nq = len(queries) if nq is None else nq
    arrays = [(ps.II_FilterChild * max(1, len(cs)))(*[ps.II_FilterChild(l, s, m) for l, s, m in cs]) for cs in queries]
    pp = (C.c_void_p * max(1, len(queries)))(*[C.cast(a, C.c_void_p) for a in arrays])
    counts = (C.c_size_t * max(1, len(queries)))(*[len(cs) for cs in queries])
    out = (C.c_void_p * max(1, len(queries)))()
    built = C.c_size_t(7)
    rc = ps.lib().II_IntersectFilterBatchDevice(nq, None if "children" in null else pp, None if "counts" in null else counts, None,
                                                None if "out" in null else out, C.byref(built))
    return rc, list(out), built.value


def test_refusals_return_minus_one_with_no_launch():
    """Every refusal happens before anything is enqueued: the child addresses are never read (they point nowhere here)"""
    ps = _ps()
    A, B = 0x1000, 0x2000  # never dereferenced
    ok = [(A, None, 0)]
    cases = [
        [ok, [(A, None, 0)] * 33],                    # more than 32 children
        [ok, [(A, None, 1), (None, B, 1)]],           # no required child
        [ok, []],                                     # no child at all
        [ok, [(A, None, 2)]],                         # OPTIONAL
        [ok, [(A, None, 0), (None, B, -1)]],          # an unknown mode
        [ok, [(A, B, 0)]],                            # both a list and a set
    ]
    ps.stats(reset=True)
    for queries in cases:
        rc, out, built = _raw_call(queries)
        assert rc == -1 and not any(out) and built == 0, queries
    for null in ("children", "counts", "out"):
        assert _raw_call([ok], null=(null,))[0] == -1, null
    assert ps.stats(reset=True).kernel_launches == 0
    # nothing to build: no set, no launch, no device needed
    assert _raw_call([[(None, None, 0)], [(None, None, 0), (A, None, 1)]]) == (0, [None, None], 0)
    assert _raw_call([], nq=0)[0] == 0


# ------------------------------------------------------------------------------------------------
# GPU helpers: children with their model (docIds, num_estimated, sort weight, tag)
# ------------------------------------------------------------------------------------------------
class Child:
    """One child of a query and what it must count as: docIds, num_estimated, sort weight (IntoChild's), result tag"""

    def __init__(self, obj, docs, est, weight=1.0, tag=4):
        self.obj, self.docs, self.est, self.weight, self.tag = obj, np.asarray(docs, dtype=np.uint64), int(est), weight, tag


def _model(children):
    """(docIds, num_estimated, child order) of the AND of [(Child or None, mode)]"""
    req = [c.docs for c, m in children if m == 0]
    docs = req[0]
    for d in req[1:]:
        docs = np.intersect1d(docs, d)
    for c, m in children:
        if m == 1 and c is not None:
            docs = np.setdiff1d(docs, c.docs)
    est = min(c.est for c, m in children if m == 0)
    keys = [2.0**62 if m else float(c.est) * c.weight for c, m in children]
    order = sorted(range(len(children)), key=lambda i: keys[i])  # stable
    return docs, est, order


def _words(ptr, n):
    """n u32 of device memory (ordered after the legacy default stream's work)"""
    import torch

    class _View:
        def __init__(self):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (int(ptr), False), "version": 3}

    return torch.as_tensor(_View(), device="cuda").cpu().numpy().view(np.uint32).copy()


def _from_device_view(rs):
    """II_PostingList_FromDevice over a settled set's docIds (freqs 1)"""
    import torch

    ps = _ps()
    m = len(rs)
    ones = torch.ones(max(m, 1), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    return ps.PostingList(ps.lib().II_PostingList_FromDevice(ps.lib().II_ResultSet_DeviceDocIds(rs.h), ones.data_ptr(), m))


def assert_query(res, children, what):
    """res = (set, docIds ptr, count ptr, cap) of one query, children = [(Child or None, mode)]"""
    ps = _ps()
    rs, d_ids, d_len, cap = res
    if any(m == 0 and (c is None or len(c.docs) == 0 and isinstance(c.obj, ps.PostingList)) for c, m in children):
        assert rs is None and cap == 0, what
        return None
    want, est, order = _model(children)
    assert rs is not None and d_ids and d_len, what
    n = len(children)
    words = _words(d_len, 2 + n)  # read before any accessor settles the set
    m = len(rs)
    assert m == len(want) and words[0] == m, what
    ids = rs.fetch(want_freqs=False)[0]
    assert ids.tolist() == want.tolist(), what
    assert cap == min(len(c.obj) if isinstance(c.obj, ps.PostingList) else ps.lib().II_ResultSet_Capacity(c.obj.h)
                      for c, md in children if md == 0), what
    assert words[1] == est, (what, words[1], est)
    assert [int(words[2 + i]) for i, (c, md) in enumerate(children) if md == 0] == [c.est for c, md in children if md == 0], what
    assert rs.child_order().tolist() == order, what
    assert ps.lib().II_ResultSet_NumChildren(rs.h) == n
    # II_IntersectEx over the same lists plus a FromDevice view of every set (empty children: an empty list)
    views = []
    for c, _ in children:
        if c is None:
            views.append(ps.PostingList.from_arrays([], []))
        elif isinstance(c.obj, ps.PostingList):
            views.append(c.obj)
        else:
            views.append(_from_device_view(c.obj))
    ex = ps.intersect_ex(views, [md for _, md in children])
    assert ex.fetch(want_freqs=False)[0].tolist() == want.tolist(), what
    return ids


_CACHE = {}


def _pool(universe=12_000, n=160):
    from test_hybrid_filter_batch import zipf_pool

    return zipf_pool(universe=universe, n=n)


def _leaves(n_docs, n_leaves=12, seed=7):
    from test_hybrid_filter_batch import cached_leaves

    return cached_leaves(n_docs, n_leaves, seed)


def _numeric_est(n_arrays, picks, lo, hi, li, hi_):
    """num_estimated of a numeric set: the sum over its leaves of the documents with a value in range"""
    from test_hybrid_filter_batch import in_range

    return sum(len(np.unique(n_arrays[j][0][in_range(n_arrays[j][1], lo, hi, li, hi_)])) for j in picks)


class Sets:
    """Pending children built on the device: ORs (quick and full), numeric ranges and II_IntersectBatchDevice ANDs, with models"""

    def __init__(self, rng, universe, n_or=8, n_num=8, n_and=4, stream=None, settle=False):
        from test_hybrid_filter_batch import numeric_model, numeric_queries

        ps = _ps()
        arrays, pool = _pool(universe)
        self.terms = [Child(pool[j], arrays[j][0], pool[j].num_estimated()) for j in range(len(pool))]
        n_arrays, leaves, prices = _leaves(universe)
        self.ors = []
        for quick in (True, False):
            picks = [rng.choice(len(pool), int(rng.integers(2, 30)), replace=False).tolist() for _ in range(n_or // 2)]
            res = ps.union_batch_device([[pool[j] for j in p] for p in picks], quick_exit=quick, stream=stream)
            for p, r in zip(picks, res):
                self.ors.append(Child(r[0], np.unique(np.concatenate([arrays[j][0] for j in p])), sum(len(arrays[j][0]) for j in p), 1.0, 1))
        qs = [q for q in numeric_queries(rng, prices, len(leaves), 6 * n_num) if q[1] <= q[2] and q[1] != 1e12][:n_num]
        res = ps.numeric_filter_batch_device([([leaves[j] for j in p], lo, hi, li, hi_) for p, lo, hi, li, hi_ in qs], stream=stream)
        self.nums = [Child(r[0], numeric_model([n_arrays[j] for j in p], lo, hi, li, hi_), _numeric_est(n_arrays, p, lo, hi, li, hi_), 1.0, 1)
                     for (p, lo, hi, li, hi_), r in zip(qs, res)]
        picks = [rng.choice(len(pool) // 4, int(rng.integers(2, 4)), replace=False).tolist() for _ in range(n_and)]
        res = ps.intersect_batch_device([[pool[j] for j in p] for p in picks], stream=stream)
        self.ands = []
        for p, r in zip(picks, res):
            docs = arrays[p[0]][0]
            for j in p[1:]:
                docs = np.intersect1d(docs, arrays[j][0])
            self.ands.append(Child(r[0], docs, min(len(arrays[j][0]) for j in p), 1.0 / len(p), 2))
        assert all(c.obj is not None for c in self.ors + self.nums + self.ands)
        if settle:
            for c in self.ors + self.nums + self.ands:
                len(c.obj)


def _shapes(S, rng):
    """the query shapes of the parity test, as functions of an rng"""
    t = lambda: S.terms[int(rng.integers(0, 24))]  # noqa: E731  (frequent terms)
    pick = lambda xs: xs[int(rng.integers(0, len(xs)))]  # noqa: E731
    quick_or = lambda: pick(S.ors[: len(S.ors) // 2])  # noqa: E731
    full_or = lambda: pick(S.ors[len(S.ors) // 2:])  # noqa: E731
    return [
        ("term-and-quick-or", lambda: [(t(), 0), (quick_or(), 0)]),
        ("term-and-full-or", lambda: [(t(), 0), (full_or(), 0)]),
        ("term-and-numeric", lambda: [(t(), 0), (pick(S.nums), 0)]),
        ("or-and-numeric", lambda: [(pick(S.ors), 0), (pick(S.nums), 0)]),
        ("term-term-numeric", lambda: [(t(), 0), (t(), 0), (pick(S.nums), 0)]),
        ("term-not-or", lambda: [(t(), 0), (pick(S.ors), 1)]),
        ("term-not-numeric", lambda: [(t(), 0), (pick(S.nums), 1)]),
        ("and-set-child", lambda: [(pick(S.ands), 0), (pick(S.ors), 0)]),
        ("or-numeric-not-or", lambda: [(pick(S.ors), 0), (pick(S.nums), 0), (pick(S.ors), 1)]),
    ]


def _call(queries, stream=None):
    return _ps().intersect_filter_batch_device([[(c.obj if c is not None else None, m) for c, m in q] for q in queries], stream=stream)


# ------------------------------------------------------------------------------------------------
# GPU: parity
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("settled", [False, True], ids=["pending", "settled"])
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_filter_and_batch_equals_intersect_ex(nq, settled):
    """Every shape on every query; the sets are shared by several queries when nq > 1"""
    rng = np.random.default_rng(nq * 2 + settled)
    S = Sets(rng, 12_000, settle=settled)
    shapes = _shapes(S, rng)
    queries, names = [], []
    for q in range(nq):
        name, make = shapes[(q + nq) % len(shapes)]
        queries.append(make())
        names.append(name)
    res = _call(queries)
    seen = set()
    for q in range(nq):
        assert_query(res[q], queries[q], (nq, q, names[q]))
        seen.add(names[q])
    assert nq == 1 or seen == {n for n, _ in shapes}


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_output_is_a_child_of_a_second_call(nq):
    """`@a (@b @tag:{x|y})`: the inner ANDs (some with an estimate on the device) as pending children of the outer ones"""
    rng = np.random.default_rng(100 + nq)
    S = Sets(rng, 12_000)
    shapes = _shapes(S, rng)
    inner = [shapes[q % len(shapes)][1]() for q in range(nq)]
    res1 = _call(inner)
    kids = []
    for q in range(nq):
        docs, est, _ = _model(inner[q])
        kids.append(Child(res1[q][0], docs, est, 1.0 / len(inner[q]), 2))
    outer = [[(S.terms[int(rng.integers(0, 40))], 0), (kids[q], 0)] + ([(S.nums[q % len(S.nums)], 1)] if q % 2 else []) for q in range(nq)]
    res2 = _call(outer)
    for q in range(nq):
        assert_query(res2[q], outer[q], ("outer", q))
        assert_query(res1[q], inner[q], ("inner", q))


@pytest.mark.gpu
def test_edge_children():
    ps = _ps()
    rng = np.random.default_rng(5)
    S = Sets(rng, 12_000)
    arrays, pool = _pool()
    n_arrays, leaves, prices = _leaves(12_000)
    from test_hybrid_filter_batch import numeric_model

    empty = Child(ps.PostingList.from_arrays([], []), [], 0)
    # a 0.1 % range over every leaf: a capacity far above its count, as the driver and as a probed child
    fin = np.sort(prices[np.isfinite(prices)])
    lo, hi = float(fin[len(fin) // 2]), float(fin[len(fin) // 2 + len(fin) // 1000])
    every = list(range(len(leaves)))
    narrow_rs = ps.numeric_filter_batch_device([([leaves[j] for j in every], lo, hi, 1, 1)])[0][0]
    narrow = Child(narrow_rs, numeric_model([n_arrays[j] for j in every], lo, hi, 1, 1), _numeric_est(n_arrays, every, lo, hi, 1, 1), 1.0, 1)
    assert ps.lib().II_ResultSet_Capacity(narrow_rs.h) > 100 * len(narrow.docs)
    every_rs = ps.numeric_filter_batch_device([([leaves[j] for j in every], -np.inf, np.inf, 1, 1)])[0][0]
    every_num = Child(every_rs, numeric_model([n_arrays[j] for j in every], -np.inf, np.inf, 1, 1),
                      _numeric_est(n_arrays, every, -np.inf, np.inf, 1, 1), 1.0, 1)
    big_or = max(S.ors, key=lambda c: len(c.docs))
    small_term = S.terms[-1]  # a short list: the list drives
    small_rs = ps.union_batch_device([[pool[150], pool[151]]], quick_exit=True)[0][0]  # a short OR: the set drives
    small_or = Child(small_rs, np.union1d(arrays[150][0], arrays[151][0]), len(arrays[150][0]) + len(arrays[151][0]), 1.0, 1)
    assert ps.lib().II_ResultSet_Capacity(small_rs.h) < len(S.terms[0].docs)
    edge_lo = Child(ps.PostingList.from_arrays([1, 2, 5, 9, U32_MAX_ID]), [1, 2, 5, 9, U32_MAX_ID], 5)
    edge_hi = Child(ps.PostingList.from_arrays([1, 9, 77, U32_MAX_ID]), [1, 9, 77, U32_MAX_ID], 4)
    wide = [(S.terms[j], 0) for j in range(20)] + [(S.ors[j % len(S.ors)], 0 if j % 3 else 1) for j in range(6)] + \
           [(S.nums[j], j % 2) for j in range(6)]
    assert len(wide) == 32
    queries = [
        [(S.terms[0], 0), (None, 0)],                       # an empty required child: no set
        [(S.terms[0], 0), (empty, 0)],                      # an empty required list: no set
        [(S.terms[0], 0), (None, 1), (empty, 1)],           # empty NOT children exclude nothing
        [(big_or, 0), (small_term, 0)],                     # a list driver
        [(S.terms[0], 0), (small_or, 0)],                   # a set driver
        [(narrow, 0), (every_num, 0)],                      # a driver whose capacity is far above its count (equal caps: the first)
        [(S.terms[1], 0), (narrow, 0)],
        [(S.terms[2], 0), (narrow, 1)],
        [(edge_lo, 0), (edge_hi, 0)],                       # docIds 1 and 2^32 - 2
        [(edge_lo, 0), (edge_hi, 1)],
        wide,                                               # 32 children
        [(S.ors[1], 0)],                                    # one child: the set itself
    ]
    res = _call(queries)
    for q, children in enumerate(queries):
        assert_query(res[q], children, ("edge", q))
    assert res[8][0].fetch(want_freqs=False)[0].tolist() == [1, 9, U32_MAX_ID]
    assert res[9][0].fetch(want_freqs=False)[0].tolist() == [2, 5]


# ------------------------------------------------------------------------------------------------
# GPU: end to end, no host wait, launches, lifetime
# ------------------------------------------------------------------------------------------------
def _compound_batch(rng, n_docs, nq=24, stream=None):
    """term AND tag-OR, term AND price range, tag-OR AND price range AND NOT tag-OR, built from pending sets; the filters they
    must hold; and every input (borrowed by the AND)"""
    S = Sets(rng, n_docs, stream=stream)
    queries = []
    for q in range(nq):
        t = S.terms[int(rng.integers(0, 16))]
        o, o2, nm = S.ors[q % len(S.ors)], S.ors[(q + 3) % len(S.ors)], S.nums[q % len(S.nums)]
        queries.append([[(t, 0), (o, 0)], [(t, 0), (nm, 0)], [(o, 0), (nm, 0), (o2, 1)]][q % 3])
    want = [_model(q)[0].astype(np.uint32) for q in queries]
    return S, queries, want


@pytest.mark.gpu
@pytest.mark.parametrize("k", [10, 1000])
@pytest.mark.parametrize("kind", ["f32_cos", "i8_l2", "f32_multi"])
def test_filter_ands_feed_the_device_knn_like_the_host_filters(kind, k):
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries
    from test_hybrid_filter_batch import _index, _knn_on_sets

    g, qs_all = _index(kind)
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    S, queries, want = _compound_batch(np.random.default_rng(len(kind) + k), 70_000, stream=s)
    sets = _call(queries, stream=s)
    labels, scores, counts, rc = _knn_on_sets(g, qd, k, sets, s)
    assert rc == 0
    s.synchronize()
    labels, scores, counts = labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], k, f, labels[i], scores[i], int(counts[i]), (kind, k, i))


@pytest.mark.gpu
def test_no_entry_point_waits_for_the_callers_stream():
    """With a kernel spinning on the caller's stream, the OR / range calls, this call and the KNN all return before it ends"""
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries
    from test_hybrid_filter_batch import _index, _knn_on_sets, _spin

    g, qs_all = _index("f32_cos")
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    outs = dict(out_labels=torch.empty((24, 10), dtype=torch.int64, device="cuda"),
                out_scores=torch.empty((24, 10), dtype=torch.float32, device="cuda"),
                out_counts=torch.empty(24, dtype=torch.int32, device="cuda"))
    s = torch.cuda.Stream()
    S, queries, _ = _compound_batch(np.random.default_rng(21), 70_000, stream=s)  # warm-up: pools, scratch, staging
    assert _knn_on_sets(g, qd, 10, _call(queries, stream=s), s, **outs)[3] == 0
    s.synchronize()
    outs["out_labels"].fill_(7)
    torch.cuda.synchronize()
    _spin(s, 2_000_000_000)  # ~1 s: longer than the host's own work of building the batch and its models
    S, queries, want = _compound_batch(np.random.default_rng(21), 70_000, stream=s)
    rc = _knn_on_sets(g, qd, 10, _call(queries, stream=s), s, **outs)[3]
    busy = not s.query()
    s.synchronize()
    assert rc == 0
    assert busy, "an entry point waited for the caller's stream"
    labels, scores, counts = (outs[n].cpu().numpy() for n in ("out_labels", "out_scores", "out_counts"))
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], 10, f, labels[i], scores[i], int(counts[i]), i)


@pytest.mark.gpu
def test_launches_do_not_depend_on_the_batch_size_or_the_children():
    ps = _ps()
    rng = np.random.default_rng(31)
    S = Sets(rng, 12_000)
    pool = S.terms[:24] + S.ors + S.nums
    seen = []
    for nq in (16, 256):
        for n in (2, 32):
            queries = [[(S.terms[q % 8], 0)] + [(pool[int(rng.integers(0, len(pool)))], int(j % 4 == 3)) for j in range(n - 1)]
                       for q in range(nq)]
            ps.stats(reset=True)
            res = _call(queries)
            seen.append(ps.stats(reset=True).kernel_launches)
            assert all(r[0] is not None for r in res)
            del res
    assert seen == [3] * 4, seen


@pytest.mark.gpu
def test_inputs_may_be_freed_right_after_the_call():
    """Every input set is freed from another thread while the AND is still held back, and the pool memory it gave back is asked
    for again and filled with other docIds before the AND runs; the KNN over the ANDs is still right.  The AND is held behind a
    kernel spinning on the caller's stream (II_ResultSet_FreeAfter makes the library's stream wait for it), so it is certainly
    pending across the frees; whether the pool would hand the freed blocks out again early without the AND's reader event is the
    allocator's choice, so this catches a missing wait when it does.  II_Score is refused and II_ResultSet_IntoChild gives NULL
    on an output (filter mode)."""
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries
    from test_hybrid_filter_batch import _index, _knn_on_sets, _spin

    ps = _ps()
    L = ps.lib()
    g, qs_all = _index("f32_cos")
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    s = torch.cuda.Stream()
    S, queries, want = _compound_batch(np.random.default_rng(8), 70_000, stream=s)
    torch.cuda.synchronize()
    _spin(s, 2_000_000_000)  # ~1 s
    hold = _call([[(S.terms[0], 0)]])[0][0]
    hold.free_after(s)  # this thread's library stream now waits for the spin
    sets = _call(queries, stream=s)  # enqueued behind it
    inputs = [c.obj for c in S.ors + S.nums + S.ands]
    for c in S.ors + S.nums + S.ands:
        c.obj = None
    caps = [L.II_ResultSet_Capacity(rs.h) for rs in inputs]
    junk = []

    def free_and_reuse():
        for rs in inputs:
            rs.close()
        inputs.clear()
        for cap in caps:  # blocks of the sizes just freed (docIds, and scores at twice the size), holding docIds no filter has
            for n in (cap, 2 * cap):
                junk.append(ps.PostingList.from_arrays(np.arange(4_000_000_000, 4_000_000_000 + n, dtype=np.uint64)))

    th = threading.Thread(target=free_and_reuse)
    th.start()
    th.join()
    assert not s.query(), "the spin ended before the inputs were freed and their memory reused: the check proves nothing"
    labels, scores, counts, rc = _knn_on_sets(g, qd, 10, sets, s)
    assert rc == 0
    s.synchronize()
    labels, scores, counts = labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], 10, f, labels[i], scores[i], int(counts[i]), i)
    del junk
    rs = _call([[(S.terms[0], 0), (S.terms[1], 0)]])[0][0]
    assert len(rs) > 0
    terms = (ps.II_TermParams * 3)(*[ps.II_TermParams(1.0, 1.0, 1.0)] * 3)
    assert L.II_Score(rs.h, ps.SCORER_BM25STD, terms, 1.0, None, None, 0.0, 1) == -1
    h, rs.h = rs.h, None
    assert not L.II_ResultSet_IntoChild(h, terms, 1.0, 0)  # consumed


@pytest.mark.gpu
def test_closed_children_are_refused_not_taken_as_empty():
    ps = _ps()
    S = Sets(np.random.default_rng(9), 12_000, n_or=2, n_num=2, n_and=1)
    gone = S.ors[0].obj
    gone.close()
    with pytest.raises(ValueError):
        ps.intersect_filter_batch_device([[(S.terms[0].obj, 0), (gone, 1)]])
    closed_list = ps.PostingList.from_arrays([1, 2, 3])
    closed_list.close()
    with pytest.raises(ValueError):
        ps.intersect_filter_batch_device([[(closed_list, 0)]])
