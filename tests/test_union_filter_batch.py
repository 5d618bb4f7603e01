"""Filter-mode ORs over posting lists and pending sets on the device with no host wait: II_UnionFilterBatchDevice, alone, composed
with itself and with II_IntersectFilterBatchDevice, and feeding VecSimB200_TopKFilteredBatchDevice.

Every set must hold the docIds II_Union(quick) gives over the same lists plus II_PostingList_FromDevice of each set child, and
numpy's union1d; its count, num_estimated (DeviceLen[1]: the sum of the children's), child order (the identity) and number of
children must follow union_plan's rule for a quick union; every KNN row fed from it must equal VecSimB200_TopKFiltered on the
host-built filter, bit for bit.
"""
import ctypes as C
import os
import re
import subprocess
import threading

import numpy as np
import pytest

from test_intersect_filter_batch import Child, Sets, _model, _shapes, _words

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
    assert hasattr(ps.lib(), "II_UnionFilterBatchDevice")
    hdr = open(os.path.join(ROOT, "include", "ii_b200.h")).read()
    assert re.search(r"int\s+II_UnionFilterBatchDevice\s*\(\s*size_t nq,\s*const II_FilterChild \*const \*children,\s*"
                     r"const size_t \*n_children,\s*void \*stream,\s*II_ResultSet \*\*out,\s*size_t \*built\)\s*;", hdr)
    assert len(re.findall(r"typedef struct \{[^}]*\} II_FilterChild;", hdr)) == 1  # the AND's child struct, reused as it is
    # the prototype takes the AND's child table as it is (-Werror: any other pointer type fails to compile)
    decl = tmp_path / "decl.c"
    decl.write_text('#include <stddef.h>\n#include "%s"\n'
                    'int (*f)(size_t, const II_FilterChild *const *, const size_t *, void *, II_ResultSet **, size_t *) =\n'
                    '    II_UnionFilterBatchDevice;\n' % os.path.join(ROOT, "include", "ii_b200.h"))
    subprocess.run(["gcc", "-Werror", "-c", str(decl), "-o", str(tmp_path / "decl.o")], check=True)
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
    """II_UnionFilterBatchDevice over queries[q] = [(list address, set address, mode)]; `null` names arguments passed as NULL"""
    ps = _ps()
    nq = len(queries) if nq is None else nq
    arrays = [(ps.II_FilterChild * max(1, len(cs)))(*[ps.II_FilterChild(l, s, m) for l, s, m in cs]) for cs in queries]
    pp = (C.c_void_p * max(1, len(queries)))(*[C.cast(a, C.c_void_p) for a in arrays])
    counts = (C.c_size_t * max(1, len(queries)))(*[len(cs) for cs in queries])
    out = (C.c_void_p * max(1, len(queries)))()
    built = C.c_size_t(7)
    rc = ps.lib().II_UnionFilterBatchDevice(nq, None if "children" in null else pp, None if "counts" in null else counts, None,
                                            None if "out" in null else out, C.byref(built))
    return rc, list(out), built.value


def test_refusals_return_minus_one_with_no_launch():
    """Every refusal happens before anything is enqueued: the child addresses are never read (they point nowhere here)"""
    ps = _ps()
    A, B = 0x1000, 0x2000  # never dereferenced
    ok = [(A, None, 0)]
    cases = [
        [ok, [(A, None, 0)] * 1025],                  # more than 1024 children
        [ok, [(A, None, 0), (None, B, 1)]],           # NOT under an OR
        [ok, [(A, None, 2)]],                         # OPTIONAL
        [ok, [(A, None, 0), (None, B, -1)]],          # an unknown mode
        [ok, [(A, B, 0)]],                            # both a list and a set
        [ok, [(None, None, 1)]],                      # an empty child with a mode other than 0
    ]
    ps.stats(reset=True)
    for queries in cases:
        rc, out, built = _raw_call(queries)
        assert rc == -1 and not any(out) and built == 0, len(queries[1])
    for null in ("children", "counts", "out"):
        assert _raw_call([ok], null=(null,))[0] == -1, null
    assert ps.stats(reset=True).kernel_launches == 0
    # nothing to build: no set, no launch, no device needed
    assert _raw_call([[(None, None, 0)], [], [(None, None, 0)] * 3]) == (0, [None, None, None], 0)
    assert _raw_call([], nq=0)[0] == 0


# ------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------
def _bound(c):
    ps = _ps()
    if c is None:
        return 0
    return len(c.obj) if isinstance(c.obj, ps.PostingList) else ps.lib().II_ResultSet_Capacity(c.obj.h)


def or_model(children):
    """(docIds, num_estimated) of the OR of [Child or None]"""
    docs = [c.docs for c in children if c is not None]
    want = np.unique(np.concatenate(docs)) if docs else np.zeros(0, dtype=np.uint64)
    return want.astype(np.uint64), sum(c.est for c in children if c is not None)


_VIEWS = {}


def _view(c):
    """the list II_Union takes for a child: the list itself, an empty list, or II_PostingList_FromDevice of a set's docIds"""
    import torch

    ps = _ps()
    if c is None:
        return ps.PostingList.from_arrays([], [])
    if isinstance(c.obj, ps.PostingList):
        return c.obj
    key = id(c.obj)
    if key not in _VIEWS or _VIEWS[key][0] is not c.obj:
        m = len(c.obj)
        if m == 0:
            v = ps.PostingList.from_arrays([], [])
        else:
            ones = torch.ones(m, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            v = ps.PostingList(ps.lib().II_PostingList_FromDevice(ps.lib().II_ResultSet_DeviceDocIds(c.obj.h), ones.data_ptr(), m))
        _VIEWS[key] = (c.obj, v)
    return _VIEWS[key][1]


def assert_or(res, children, what, host_check=True):
    """res = (set, docIds ptr, count ptr, cap) of one query, children = [Child or None]"""
    ps = _ps()
    rs, d_ids, d_len, cap = res
    if all(_bound(c) == 0 for c in children):
        assert rs is None and cap == 0, what
        return None
    want, est = or_model(children)
    assert rs is not None and d_ids and d_len, what
    words = _words(d_len, 2)  # read before any accessor settles the set
    m = len(rs)
    assert m == len(want) and words[0] == m, (what, m, len(want))
    assert words[1] == min(est, 2**32 - 1), (what, words[1], est)
    ids = rs.fetch(want_freqs=False)[0]
    assert ids.tolist() == want.tolist(), what
    assert len(want) <= cap <= sum(_bound(c) for c in children), what
    assert rs.child_order().tolist() == list(range(len(children))), what
    assert ps.lib().II_ResultSet_NumChildren(rs.h) == len(children)
    if host_check:  # II_Union(quick) over the same lists plus a FromDevice view of every set
        host = ps.union([_view(c) for c in children], quick_exit=True)
        assert host.fetch(want_freqs=False)[0].tolist() == want.tolist(), what
    return ids


def _call(queries, stream=None):
    return _ps().union_filter_batch_device([[c.obj if c is not None else None for c in q] for q in queries], stream=stream)


def _and_call(queries, stream=None):
    return _ps().intersect_filter_batch_device([[(c.obj if c is not None else None, m) for c, m in q] for q in queries], stream=stream)


def _ifb_children(S, rng, n=12, stream=None):
    """outputs of II_IntersectFilterBatchDevice over S, some with their estimate still on the device (a numeric child), as Children"""
    shapes = _shapes(S, rng)
    inner = [shapes[q % len(shapes)][1]() for q in range(n)]
    res = _and_call(inner, stream=stream)
    out = []
    for q in range(n):
        if res[q][0] is None:
            continue
        docs, est, _ = _model(inner[q])
        out.append(Child(res[q][0], docs, est, 1.0 / len(inner[q]), 2))
    return out


class Kinds:
    """every kind of child: term lists, ANDs (II_IntersectBatchDevice), quick and full ORs, numeric sets, filter ANDs"""

    def __init__(self, rng, universe=12_000, settle=False, stream=None):
        self.S = Sets(rng, universe, stream=stream, settle=settle)
        self.filter_ands = _ifb_children(self.S, rng, stream=stream)
        if settle:
            for c in self.filter_ands:
                len(c.obj)
        S = self.S
        self.all = S.terms[:60] + S.ands + S.ors + S.nums + self.filter_ands


def _pick(rng, kinds, n, empty_rate=0.0):
    out = []
    for _ in range(n):
        if empty_rate and rng.random() < empty_rate:
            out.append(None)
        else:
            out.append(kinds.all[int(rng.integers(0, len(kinds.all)))])
    return out


# ------------------------------------------------------------------------------------------------
# GPU: parity
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("settled", [False, True], ids=["pending", "settled"])
@pytest.mark.parametrize("n", [1, 2, 20, 21, 200, 1024])
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_union_filter_batch_equals_ii_union(nq, n, settled):
    """Children of every kind, shared across the queries and repeated inside them; II_Union(quick) is the check on every query
    of the smaller batches and on every 16th of the 256-query ones (numpy on all)"""
    rng = np.random.default_rng(nq * 10_000 + n * 2 + settled)
    K = Kinds(rng, settle=settled)
    queries = [_pick(rng, K, n) for _ in range(nq)]
    res = _call(queries)
    for q in range(nq):
        assert_or(res[q], queries[q], (nq, n, q), host_check=nq <= 16 or q % 16 == 0)


@pytest.mark.gpu
def test_deferred_estimate_is_summed_on_the_device():
    """A pending numeric set or filter AND with its estimate on the device: DeviceLen[1] holds the sum before the set settles,
    and the settled set's estimate (read by a later AND, which takes it from the host) is the same sum"""
    rng = np.random.default_rng(3)
    K = Kinds(rng)
    S = K.S
    inner = [[(S.terms[0], 0), (S.nums[4], 0)], [(S.ors[0], 0), (S.nums[5], 0)]]  # ANDs whose estimate waits for the device
    d = [Child(r[0], *_model(q)[:2], 0.5, 2) for q, r in zip(inner, _and_call(inner))]
    queries = [[S.nums[0], S.terms[1]], [S.nums[1], S.nums[2], S.ors[0]], [d[0], S.terms[2], d[1]], [S.nums[3]], [d[1], S.ands[0]]]
    res = _call(queries)
    for q in range(len(queries)):
        assert_or(res[q], queries[q], ("deferred", q))  # settles the sets
    kids = [Child(res[q][0], *or_model(queries[q]), 1.0, 1) for q in range(len(queries))]
    from test_intersect_filter_batch import assert_query

    outer = [[(S.terms[0], 0), (kids[q], 0)] for q in range(len(kids))]
    res2 = _and_call(outer)
    for q in range(len(outer)):
        assert_query(res2[q], outer[q], ("outer", q))


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 16, 256])
def test_three_level_trees(nq):
    """`@tag:{sale} ((@a @b) | @c)`: ANDs, an OR over them, an AND over the OR; and an OR over ORs; all pending"""
    from test_intersect_filter_batch import assert_query

    rng = np.random.default_rng(200 + nq)
    K = Kinds(rng)
    S = K.S
    shapes = _shapes(S, rng)
    inner = [shapes[q % len(shapes)][1]() for q in range(2 * nq)]
    r1 = _and_call(inner)
    ands = []
    for q in range(2 * nq):
        docs, est, _ = _model(inner[q])
        ands.append(Child(r1[q][0], docs, est, 1.0 / len(inner[q]), 2) if r1[q][0] is not None else None)
    ors_q = [[ands[2 * q], ands[2 * q + 1], S.terms[q % 40]] for q in range(nq)]
    r2 = _call(ors_q)
    ors = [Child(r2[q][0], *or_model(ors_q[q]), 1.0, 1) for q in range(nq)]
    top_q = [[(S.terms[int(rng.integers(0, 8))], 0), (ors[q], 0)] for q in range(nq)]
    r3 = _and_call(top_q)
    oo_q = [[ors[q], ors[(q + 1) % nq], S.nums[q % len(S.nums)]] for q in range(nq)]
    r4 = _call(oo_q)
    for q in range(nq):
        assert_query(r3[q], top_q[q], ("and-over-or", q))
        assert_or(r4[q], oo_q[q], ("or-over-or", q), host_check=q % 16 == 0)
        assert_or(r2[q], ors_q[q], ("or-over-and", q), host_check=q % 16 == 0)


@pytest.mark.gpu
def test_edge_children():
    ps = _ps()
    from test_hybrid_filter_batch import numeric_model
    from test_intersect_filter_batch import _leaves, _numeric_est

    rng = np.random.default_rng(5)
    K = Kinds(rng)
    S = K.S
    n_arrays, leaves, prices = _leaves(12_000)
    empty = Child(ps.PostingList.from_arrays([], []), [], 0)
    fin = np.sort(prices[np.isfinite(prices)])
    lo, hi = float(fin[len(fin) // 2]), float(fin[len(fin) // 2 + len(fin) // 1000])
    every = list(range(len(leaves)))
    narrow_rs = ps.numeric_filter_batch_device([([leaves[j] for j in every], lo, hi, 1, 1)])[0][0]
    narrow = Child(narrow_rs, numeric_model([n_arrays[j] for j in every], lo, hi, 1, 1), _numeric_est(n_arrays, every, lo, hi, 1, 1), 1.0, 1)
    assert ps.lib().II_ResultSet_Capacity(narrow_rs.h) > 100 * len(narrow.docs)
    # docIds 1 and 2^32 - 2 in every kind of set
    a = ps.PostingList.from_arrays([1, 2, 5, 9, U32_MAX_ID])
    b = ps.PostingList.from_arrays([1, 9, 77, U32_MAX_ID])
    la, lb = Child(a, [1, 2, 5, 9, U32_MAX_ID], 5), Child(b, [1, 9, 77, U32_MAX_ID], 4)
    e_and = Child(ps.intersect_batch_device([[a, b]])[0][0], [1, 9, U32_MAX_ID], 4, 0.5, 2)
    e_or = Child(ps.union_batch_device([[a, b]], quick_exit=True)[0][0], [1, 2, 5, 9, 77, U32_MAX_ID], 9, 1.0, 1)
    e_full = Child(ps.union_batch_device([[a, b]], quick_exit=False)[0][0], [1, 2, 5, 9, 77, U32_MAX_ID], 9, 1.0, 1)
    e_ifb = Child(_and_call([[(la, 0), (lb, 0)]])[0][0], [1, 9, U32_MAX_ID], 4, 0.5, 2)
    e_none = Child(ps.intersect_batch_device([[a, ps.PostingList.from_arrays([3, 4])]])[0][0], [], 2, 0.5, 2)  # disjoint bounds
    w = ps.IndexWriter(numeric=True)
    for d, v in ((1, 5.0), (U32_MAX_ID, 6.0)):
        w.add_numeric(d, v)
    leaf = ps.NumericList(w.blocks())
    e_num = Child(ps.numeric_filter_batch_device([([leaf], 0.0, 10.0, 1, 1)])[0][0], [1, U32_MAX_ID], 2, 1.0, 1)
    same = S.ors[0]
    queries = [
        [None],                                         # every child empty: no set
        [None, empty],
        [None, S.terms[0], empty],                      # empty children next to a list
        [same, same, same],                             # the same set repeated
        [narrow],                                       # a capacity 100 times the count
        [narrow, S.terms[3]],
        [e_and, e_or, e_full, e_ifb, e_num],            # docIds 1 and 2^32 - 2 in sets of every kind
        [e_and, la],
        [e_num, S.terms[5]],                            # a window from 1 to 2^32 - 2
        [e_none],                                       # an AND whose bounds exclude each other: a set with nothing in it
        [e_none, S.terms[6]],
    ]
    res = _call(queries)
    for q, children in enumerate(queries):
        assert_or(res[q], children, ("edge", q))
    assert res[6][0].fetch(want_freqs=False)[0].tolist() == [1, 2, 5, 9, 77, U32_MAX_ID]
    assert res[9][0] is not None and len(res[9][0]) == 0


@pytest.mark.gpu
def test_window_bounds_follow_the_children():
    """256 ORs over pending ANDs whose docIds all lie in [4.0e9, 4.0e9 + 1e5]: each window spans that range, not docIds from 0
    (which would take about 128 GB of bitmap for the batch)"""
    ps = _ps()
    rng = np.random.default_rng(11)
    base = 4_000_000_000
    arrays = [np.unique(rng.integers(base, base + 100_000, int(rng.integers(2_000, 40_000)))).astype(np.uint64) for _ in range(48)]
    lists = [ps.PostingList.from_arrays(a) for a in arrays]
    picks = [rng.choice(48, 2, replace=False).tolist() for _ in range(128)]
    ands = ps.intersect_batch_device([[lists[i] for i in p] for p in picks])
    kids = [Child(r[0], np.intersect1d(arrays[p[0]], arrays[p[1]]), min(len(arrays[i]) for i in p), 0.5, 2) for p, r in zip(picks, ands)]
    queries = [[kids[q % 128], kids[(q * 7 + 3) % 128], kids[(q * 13 + 5) % 128]] for q in range(256)]
    res = _call(queries)
    for q in range(256):
        assert_or(res[q], queries[q], ("window", q), host_check=q % 32 == 0)


# ------------------------------------------------------------------------------------------------
# GPU: end to end, no host wait, launches, lifetime
# ------------------------------------------------------------------------------------------------
def _or_batch(rng, n_docs, nq=24, stream=None):
    """(term ∧ tag) | (term ∧ tag), range | range, (tag ∧ range) | term over pending sets; the filters they must hold; the inputs"""
    S = Sets(rng, n_docs, stream=stream)
    inner = []
    for q in range(nq):
        t, t2 = S.terms[int(rng.integers(0, 16))], S.terms[int(rng.integers(0, 16))]
        o, o2, nm = S.ors[q % len(S.ors)], S.ors[(q + 3) % len(S.ors)], S.nums[q % len(S.nums)]
        inner += [[(t, 0), (o, 0)], [(t2, 0), (o2, 0)], [(o, 0), (nm, 0)]]
    r1 = _and_call(inner, stream=stream)
    ands = [Child(r[0], *_model(q)[:2], 0.5, 2) for q, r in zip(inner, r1)]
    queries = []
    for q in range(nq):
        nm, nm2 = S.nums[q % len(S.nums)], S.nums[(q + 1) % len(S.nums)]
        queries.append([[ands[3 * q], ands[3 * q + 1]], [nm, nm2], [ands[3 * q + 2], S.terms[int(rng.integers(0, 16))]]][q % 3])
    want = [or_model(q)[0].astype(np.uint32) for q in queries]
    return S, ands, queries, want


@pytest.mark.gpu
@pytest.mark.parametrize("k", [10, 1000])
@pytest.mark.parametrize("kind", ["f32_cos", "i8_l2", "f32_multi"])
def test_filter_ors_feed_the_device_knn_like_the_host_filters(kind, k):
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries
    from test_hybrid_filter_batch import _index, _knn_on_sets

    g, qs_all = _index(kind)
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    S, ands, queries, want = _or_batch(np.random.default_rng(len(kind) + k), 70_000, stream=s)
    sets = _call(queries, stream=s)
    labels, scores, counts, rc = _knn_on_sets(g, qd, k, sets, s)
    assert rc == 0
    s.synchronize()
    labels, scores, counts = labels.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    for i, f in enumerate(want):
        assert_row_equals_filtered(g, qs[i], k, f, labels[i], scores[i], int(counts[i]), (kind, k, i))


@pytest.mark.gpu
def test_no_entry_point_waits_for_the_callers_stream():
    """With a kernel spinning on the caller's stream, the child calls, this call and the KNN all return before it ends"""
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
    S, ands, queries, _ = _or_batch(np.random.default_rng(21), 70_000, stream=s)  # warm-up: pools, scratch, staging
    assert _knn_on_sets(g, qd, 10, _call(queries, stream=s), s, **outs)[3] == 0
    s.synchronize()
    outs["out_labels"].fill_(7)
    torch.cuda.synchronize()
    _spin(s, 2_000_000_000)  # ~1 s: longer than the host's own work of building the batch and its models
    S, ands, queries, want = _or_batch(np.random.default_rng(21), 70_000, stream=s)
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
    K = Kinds(rng)
    seen = []
    for nq in (16, 256):
        for n in (2, 200):
            queries = [_pick(rng, K, n) for _ in range(nq)]
            ps.stats(reset=True)
            res = _call(queries)
            seen.append(ps.stats(reset=True).kernel_launches)
            assert all(r[0] is not None for r in res)
            del res
    assert seen == [4] * 4, seen


@pytest.mark.gpu
def test_list_only_batches_are_unchanged():
    """II_UnionBatchDevice(quick) over lists: the same sets and launches as II_Union; the new call over the same lists gives the
    same docIds, capacity and estimate in the same 4 launches"""
    from test_hybrid_filter_batch import _host_union, assert_same_set, zipf_pool

    ps = _ps()
    arrays, pool = zipf_pool()
    rng = np.random.default_rng(17)
    picks = [rng.choice(len(pool), int(rng.integers(1, 60)), replace=False).tolist() for _ in range(32)]
    batch = [[pool[j] for j in p] for p in picks]
    ps.stats(reset=True)
    res = ps.union_batch_device(batch, quick_exit=True)
    assert ps.stats(reset=True).kernel_launches == 4
    res2 = ps.union_filter_batch_device(batch)
    assert ps.stats(reset=True).kernel_launches == 4
    L = ps.lib()
    for i, p in enumerate(picks):
        host = _host_union(batch[i], True)
        assert_same_set(res[i][0], host, True, what=i)
        kids = [Child(pool[j], arrays[j][0], pool[j].num_estimated()) for j in p]
        assert_or(res2[i], kids, ("lists", i))
        assert L.II_ResultSet_Capacity(res2[i][0].h) == L.II_ResultSet_Capacity(host.h)


@pytest.mark.gpu
def test_inputs_may_be_freed_right_after_the_call():
    """Every input set is freed from another thread while the OR is held behind a kernel spinning on the caller's stream, and the
    pool memory it gave back is asked for again and filled with other docIds; the KNN over the ORs is still right.  II_Score is
    refused and II_ResultSet_IntoChild gives NULL on an output (filter mode)."""
    import torch
    from test_hybrid_device_batch import _dev, assert_row_equals_filtered, stored_queries
    from test_hybrid_filter_batch import _index, _knn_on_sets, _spin

    ps = _ps()
    L = ps.lib()
    g, qs_all = _index("f32_cos")
    qs = qs_all[:24]
    qd = _dev(stored_queries(g, qs))
    s = torch.cuda.Stream()
    S, ands, queries, want = _or_batch(np.random.default_rng(8), 70_000, stream=s)
    torch.cuda.synchronize()
    _spin(s, 2_000_000_000)  # ~1 s
    hold = _call([[S.terms[0]]])[0][0]
    hold.free_after(s)  # this thread's library stream now waits for the spin
    sets = _call(queries, stream=s)  # enqueued behind it
    kids = S.ors + S.nums + S.ands + ands
    inputs = [c.obj for c in kids]
    for c in kids:
        c.obj = None
    caps = [L.II_ResultSet_Capacity(rs.h) for rs in inputs]
    junk = []

    def free_and_reuse():
        for rs in inputs:
            rs.close()
        inputs.clear()
        for cap in caps:  # blocks of the sizes just freed, holding docIds no filter has
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
    rs = _call([[S.terms[0], S.terms[1]]])[0][0]
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
        ps.union_filter_batch_device([[S.terms[0].obj, gone]])
    closed_list = ps.PostingList.from_arrays([1, 2, 3])
    closed_list.close()
    with pytest.raises(ValueError):
        ps.union_filter_batch_device([[closed_list]])
    # a list carrying a nested set (II_ResultSet_IntoChild) is refused, as by II_UnionBatchDevice, with no launch
    nested = ps.union([S.terms[0].obj, S.terms[1].obj]).into_child([(1.0, 1.0, 1.0)] * 2)
    ps.stats(reset=True)
    with pytest.raises(ValueError):
        ps.union_filter_batch_device([[S.terms[2].obj], [S.terms[0].obj, nested]])
    assert ps.stats(reset=True).kernel_launches == 0
