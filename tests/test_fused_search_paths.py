"""The fused AND batch search (II_SearchTopNBatch: fused_itemq_kernel, fused_window_kernel, fused_and_kernel<2|3|4|8>,
fused_topn_kernel) held to the oracle on every membership path, at its edges and through the top-N folds.

The CPU half restates in Python what the host and the kernels decide for each query and each driver chunk: the aggregate
child order (a stable sort by num_estimated; its first list drives), the chunking, the two window lower bounds of
fused_window_kernel, the all-fit / list-by-list / pivot-bucket choice of fused_and_kernel, the pivot bucket of every driver
entry, the per-chunk survivors and the launch split at kMaxCand.  It reads the constants those decisions rest on from the
sources, so a change of one fails here instead of silently leaving a class untested, and it asserts that the fixtures below
reach every class.

The GPU half runs those fixtures through II_SearchTopNBatch and compares each reply with the oracle directly: docIds from a
numpy intersection, every hit scored by oracle/scorer_oracle.c with the freqs in aggregate order and GetSlop = children - 1
(the lists carry no positions), replies ranked (score desc, docId asc).  The kernel launch count proves the fused path
answered: a failed fused batch falls back to the per-query chains and would otherwise pass unnoticed.
"""
import os
import re
from functools import reduce

import numpy as np
import pytest

import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "redisearch_b200", "csrc")

# restated from the sources; test_constants_match_the_sources pins every one
II_THREADS, II_ITEMS, CHUNK, SMEM_ELEMS = 256, 4, 1024, 8192
MAX_LISTS, MAX_TOPN = 8, 128
PIVOTS = 2048
TOPN_TILE, TOPN_PER_THREAD = 1024, 4
MAX_CAND = 96 << 20

TOP_NS = (1, 7, 10, 100, 127, 128)
N_DOCS = 3_000_000
AGG_WEIGHT = 0.7
WEIGHTS = (1.0, 0.5, 1.5, 0.3, 1.25, 0.75, 1.1, 0.9)


def agg_weight(scorer):
    """BM25STD.TANH at 0.1: its scores then stay clear of tanh's saturation, where distinct scores crowd within 1e-12"""
    return 0.1 if scorer == ol.SCORER_BM25STD_TANH else AGG_WEIGHT


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_constants_match_the_sources():
    h, cu, host = _read("ii_kernels.h"), _read("ii_kernels.cu"), _read("ii_host.cpp")

    def const(text, name):
        m = re.search(r"\b" + name + r"\s*=\s*(\d+)\s*[;,]", text)
        assert m, name
        return int(m.group(1))

    assert const(h, "kIIThreads") == II_THREADS and const(h, "kIIItems") == II_ITEMS
    assert re.search(r"\bkIIChunk\s*=\s*kIIThreads\s*\*\s*kIIItems\s*;", h) and II_THREADS * II_ITEMS == CHUNK
    assert const(h, "kIISmemElems") == SMEM_ELEMS
    assert const(h, "kFusedMaxLists") == MAX_LISTS and const(h, "kFusedMaxTopN") == MAX_TOPN
    assert const(cu, "kPivots") == PIVOTS
    topn = cu[cu.index("fused_topn_kernel("):]
    assert const(topn, "kTile") == TOPN_TILE and const(topn, "kPerThread") == TOPN_PER_THREAD
    m = re.search(r"\bkMaxCand\s*=\s*\(size_t\)\s*(\d+)\s*<<\s*(\d+)\s*;", host)
    assert m and int(m.group(1)) << int(m.group(2)) == MAX_CAND


# ------------------------------------------------------------------------------------------------
# the host's and the kernels' decisions, restated
# ------------------------------------------------------------------------------------------------
class Term:
    """One child: its docIds and freqs after any field-mask filter, and num_estimated (the unfiltered count)."""

    def __init__(self, name, ids, freqs, estimated=None):
        self.name, self.ids, self.freqs = name, np.asarray(ids, dtype=np.int64), np.asarray(freqs, dtype=np.uint32)
        self.estimated = len(self.ids) if estimated is None else estimated


def aggregate_order(terms):
    """intersection.rs:110-145: a stable sort ascending by num_estimated (Python's sort is stable)"""
    return sorted(range(len(terms)), key=lambda t: terms[t].estimated)


def n_chunks(n):
    return (n + CHUNK - 1) // CHUNK


def driver_chunks(terms):
    """fused_batch: work items of a query = chunks of the list at order[0], the driver"""
    return n_chunks(len(terms[aggregate_order(terms)[0]].ids))


def launch_split(chunks_per_query, top_n):
    """fused_batch: queries go into one launch while their candidate slots fit kMaxCand (a lone query always does)"""
    launches, items, first = 0, 0, True
    for ch in chunks_per_query:
        if not first and (items + ch) * top_n > MAX_CAND:
            launches, items = launches + 1, 0
        items += ch
        first = False
    return launches + 1


def old_sizing_items(terms):
    """what fused_batch sized the scratch from before it took the driver: the child with the fewest actual entries"""
    return n_chunks(min(len(t.ids) for t in terms))


def chunk_classes(terms, c):
    """fused_window_kernel + fused_and_kernel for driver chunk c of a query: returns a dict of the classes it reaches"""
    order = aggregate_order(terms)
    A = terms[order[0]].ids
    others = [terms[t].ids for t in order[1:]]
    start, end = c * CHUNK, min((c + 1) * CHUNK, len(A))
    doc = A[start:end]
    k_lo, k_hi = int(A[start]), int(A[end - 1]) + 1  # k_hi < 2^32: docIds are < 2^32 - 1
    wins = [(int(np.searchsorted(B, k_lo, "left")), int(np.searchsorted(B, k_hi, "left"))) for B in others]
    out = {"len": end - start, "windows": [hi - lo for lo, hi in wins], "staged": [], "pivot": [], "edges": set(), "early_exit": False}
    total, all_fit = 0, True
    for lo, hi in wins:
        all_fit = all_fit and hi - lo <= SMEM_ELEMS and total + hi - lo <= SMEM_ELEMS
        if all_fit:
            total += hi - lo
    out["mode"] = "all_fit" if all_fit else "list"
    out["total"] = total if all_fit else None
    alive = np.ones(len(doc), dtype=bool)
    for j, (B, (lo, hi)) in enumerate(zip(others, wins)):
        if not all_fit and not alive.any():
            out["early_exit"] = True  # __syncthreads_or: no entry survives, the later children are never probed
            break
        W = B[lo:hi]
        if not all_fit and hi - lo > SMEM_ELEMS:
            rng_ = hi - lo
            step = (rng_ + PIVOTS - 1) // PIVOTS
            nbuckets = (rng_ + step - 1) // step
            piv = B[lo + np.arange(nbuckets) * step]
            d = doc[alive]
            a = np.searchsorted(piv, d, "right")  # upper_bound - 1 is the bucket; a == 0: below the window
            out["pivot"].append(rng_)
            if (a == 0).any():
                out["edges"].add("below")
            if np.isin(d, piv[1:]).any():
                out["edges"].add("bucket_first")
            if (d == piv[0]).any():
                out["edges"].add("window_first")
            if (d == W[-1]).any():
                out["edges"].add("window_last")
            if (d > W[-1]).any():
                out["edges"].add("above")
        elif not all_fit:
            out["staged"].append(hi - lo)
        alive &= np.isin(doc, W)
    out["survivors"] = int(alive.sum())
    return out


def query_classes(terms):
    return [chunk_classes(terms, c) for c in range(driver_chunks(terms))]


def candidates(classes, top_n):
    """fused_and_kernel keeps min(survivors, top_n) per chunk: the query's candidate list for fused_topn_kernel"""
    return sum(min(k["survivors"], top_n) for k in classes)


# ------------------------------------------------------------------------------------------------
# fixtures (numpy only: the CPU tests show what they reach, the GPU tests run them)
# ------------------------------------------------------------------------------------------------
def stepped_freqs(rng, n, top=29):
    """freqs in 1..top whose neighbours always differ: a position off by one changes the score"""
    return (1 + np.cumsum(rng.integers(1, top, n)) % top).astype(np.uint32)


def _crafted():
    """B = the even docIds, C = multiples of 3, D = multiples of 5; A = a driver whose chunks are laid out against B"""
    rng = np.random.default_rng(2024)
    NB = 1_200_000
    B = 2 * np.arange(1, NB + 1, dtype=np.int64)
    C = 3 * np.arange(1, 800_001, dtype=np.int64)
    D = 5 * np.arange(1, 480_001, dtype=np.int64)
    chunks, s = [], 10

    def edges_chunk(W):
        # window of exactly W entries of B: A[0] = B[s] - 1 below it, A[-1] = B[s+W-1] + 1 above it, both ends of the window,
        # bucket first entries (and the entries just before them) of the pivot search, other members and non-members
        nonlocal s
        first, last = B[s], B[s + W - 1]
        step = (W + PIVOTS - 1) // PIVOTS
        nb = (W + step - 1) // step
        piv = B[s + np.arange(1, nb) * step]
        pre = B[s + np.arange(1, nb) * step - 1]
        inner = B[s + 1:s + W - 1]
        mem = np.unique(np.concatenate([rng.choice(piv[piv < last], min(300, int((piv < last).sum())), replace=False),
                                        rng.choice(pre[pre > first], min(150, int((pre > first).sum())), replace=False),
                                        rng.choice(inner, 150, replace=False)]))
        mem = mem[(mem > first) & (mem < last)]
        odd = rng.choice(B[s:s + W - 1] + 1, 1020 - len(mem), replace=False)
        chunks.append(np.sort(np.concatenate([[first - 1, first, last, last + 1], mem, odd])))
        s += W + 1

    def count_chunk(W, m, n=CHUNK):
        # n entries of which exactly m are in B
        nonlocal s
        mem = B[s:s + W] if m == W else rng.choice(B[s:s + W], m, replace=False)
        odd = rng.choice(B[s:s + W] + 1, n - m, replace=False)
        chunks.append(np.sort(np.concatenate([mem, odd])))
        s += W + 1

    def none_chunk(W):
        # no entry in B or in C: the 3-child AND (A, C, B) leaves the list-by-list loop before B
        nonlocal s
        v = np.arange(B[s] + 1, B[s + W - 1])
        chunks.append(np.sort(rng.choice(v[(v % 6 == 1) | (v % 6 == 5)], CHUNK, replace=False)))
        s += W + 1

    count_chunk(3000, 129)
    edges_chunk(2000)      # all windows fit, total < 8192
    edges_chunk(8192)      # all windows fit, total == 8192
    for m in (0, 1, 7, 10):
        count_chunk(3000, m)
    edges_chunk(8193)      # pivot path from here on (2 children)
    edges_chunk(PIVOTS * 5)
    edges_chunk(PIVOTS * 5 + 1)
    none_chunk(9000)
    for m in (100, 127, 128):
        count_chunk(3000, m)
    count_chunk(CHUNK, CHUNK)  # every entry survives: the CTA sorts 1024
    for _ in range(9):
        count_chunk(3000, 600)
    edges_chunk(1_050_000)
    count_chunk(2000, 150, n=300)  # partial last chunk
    assert s <= NB
    A = np.concatenate(chunks)
    assert (np.diff(A) > 0).all() and len(A) == 25 * CHUNK + 300
    ids = {"A": A, "B": B, "C": C, "D": D}
    for n in (1, 1023, 1024, 1025):
        ids[f"L{n}"] = np.sort(rng.choice(2_400_000, n, replace=False) + 1)
    # the random corpus: 8 lists sharing 4,000 docIds, for the 4- and 8-child instantiations
    shared = rng.choice(N_DOCS - 10, 4000, replace=False) + 1
    for k, size in enumerate((6_000, 12_000, 25_000, 40_000, 60_000, 90_000, 120_000, 200_000)):
        ids[f"R{k}"] = np.union1d(shared, rng.choice(N_DOCS - 10, size, replace=False) + 1)
    return {name: Term(name, v, stepped_freqs(rng, len(v))) for name, v in ids.items()}


def _extreme():
    """docIds 1 and 0xFFFFFFFE at both ends of the driver and of the children: the last chunk's k_hi is 0xFFFFFFFF"""
    rng = np.random.default_rng(77)
    top = 0xFFFFFFFE

    def mk(n, keep):
        mid = rng.choice(np.arange(2, 60_000, dtype=np.int64), n, replace=False)
        high = top - 1 - rng.choice(60_000, n // 2, replace=False)
        return np.unique(np.concatenate([[1, top], mid, high, keep]))

    common = np.concatenate([rng.choice(np.arange(2, 60_000), 300, replace=False), top - 1 - rng.choice(60_000, 300, replace=False)])
    ids = {"X": mk(800, common), "Y": mk(20_000, common), "Z": mk(30_000, common)}
    return {name: Term(name, v, stepped_freqs(rng, len(v))) for name, v in ids.items()}


def _masked():
    """Field-mask-filtered children keep num_estimated = the unfiltered count (II_PostingList_FromBlocks): the aggregate
    order by estimate then differs from the order by length.  raw = every posting written, kept = what the filter keeps."""
    rng = np.random.default_rng(31)
    out = {}
    U = np.sort(rng.choice(400_000, 100_000, replace=False) + 1)
    U2 = np.sort(rng.choice(400_000, 20_000, replace=False) + 1)
    U3 = np.union1d(U2[::2], rng.choice(400_000, 50_000, replace=False) + 1)
    # M1 (FreqsFields): 150,000 postings, 2,000 kept, half of them in U;  M2 (FreqsFieldsWide, a mask bit above 63): 120,000
    # postings, 3,000 kept, mostly in U2 and U3
    for name, raw_n, kept_from, n_kept in (("M1", 150_000, U, 2_000), ("M2", 120_000, np.intersect1d(U2, U3), 3_000)):
        kept = np.union1d(rng.choice(kept_from, min(len(kept_from), n_kept // 2 if name == "M1" else n_kept - 400), replace=False),
                          rng.choice(400_000, n_kept // 2 if name == "M1" else 400, replace=False) + 1)
        rest = rng.permutation(np.setdiff1d(rng.choice(400_000, raw_n + 10_000, replace=False) + 1, kept))[:raw_n - len(kept)]
        raw = np.union1d(kept, rest)
        assert len(raw) == raw_n
        out[name] = (raw, stepped_freqs(rng, raw_n), np.isin(raw, kept))
    terms = {n: Term(n, v, stepped_freqs(rng, len(v))) for n, v in (("U", U), ("U2", U2), ("U3", U3))}
    for name, (raw, fr, keep) in out.items():
        terms[name] = Term(name, raw[keep], fr[keep], estimated=len(raw))
        terms[name].raw = (raw, fr, keep)
    return terms


# codec, field-mask filter, the mask of a posting the filter drops (M2's filter needs more than 64 bits: FromBlocksWideMask)
MASK_CODEC = {"M1": (ol.CODEC_FREQS_FIELDS, 0b10, 0b01), "M2": (ol.CODEC_FREQS_FIELDS_WIDE, 1 << 100, 1 << 3)}

CRAFTED_BATCHES = {  # kN of fused_and_kernel = the batch's largest child count, rounded up to 2 / 3 / 4 / 8
    2: [("A", "B"), ("A",), ("L1", "B"), ("L1023", "B"), ("L1024", "C"), ("L1025", "B")],
    3: [("A", "C", "B"), ("A", "B"), ("A",), ("L1025", "C", "B"), ("L1024", "B", "C")],
    4: [("A", "D", "C", "B"), ("A", "C", "B"), ("A", "B"), ("R0", "R3", "R5", "R7")],
    8: [tuple(f"R{k}" for k in range(8)), ("R0", "R3", "R5", "R7"), ("R1", "R2"), ("R0",), ("A", "B")],
    1: [("A",), ("R0",), ("L1025",)],  # one child everywhere: fused_window_kernel is skipped
}
EXTREME_QUERIES = [("X", "Y", "Z"), ("X", "Z"), ("X",)]
MASK_QUERIES = [("U", "M1"), ("U2", "M2", "U3"), ("M2", "U")]


@pytest.fixture(scope="module")
def crafted():
    return _crafted()


@pytest.fixture(scope="module")
def masked():
    return _masked()


def _q(corpus, names):
    return [corpus[n] for n in names]


# ------------------------------------------------------------------------------------------------
# CPU: every class is reached
# ------------------------------------------------------------------------------------------------
def test_crafted_fixtures_reach_every_membership_path_and_edge(crafted):
    ab = query_classes(_q(crafted, ("A", "B")))
    assert [k["total"] for k in ab if k["mode"] == "all_fit" and k["total"] == SMEM_ELEMS], "all-fit with exactly 8192 staged"
    assert [k for k in ab if k["mode"] == "all_fit" and 0 < k["total"] < SMEM_ELEMS]
    pivots = sorted(set(p for k in ab for p in k["pivot"]))
    for w in (SMEM_ELEMS + 1, PIVOTS * 5, PIVOTS * 5 + 1):
        assert w in pivots, (w, pivots)
    assert max(pivots) >= 1_000_000
    edges = set().union(*[k["edges"] for k in ab])
    assert edges >= {"below", "bucket_first", "window_first", "window_last", "above"}, edges
    acb = query_classes(_q(crafted, ("A", "C", "B")))
    assert [k for k in acb if k["mode"] == "list" and SMEM_ELEMS in k["staged"]], "list by list with a staged window of 8192"
    assert [k for k in acb if k["early_exit"]], "list by list with no survivor before the last child"
    assert [k for k in acb if k["mode"] == "list" and k["pivot"]]
    # driver lengths and a partial last chunk
    lens = {len(crafted[q[0]].ids) for b in CRAFTED_BATCHES.values() for q in b}
    assert {1, 1023, 1024, 1025} <= lens and len(crafted["A"].ids) % CHUNK
    for b in CRAFTED_BATCHES.values():
        for q in b:
            assert aggregate_order(_q(crafted, q))[0] == 0, q  # the fixtures name the driver first
    # every kernel instantiation, with smaller queries in the same batch
    for kn, batch in CRAFTED_BATCHES.items():
        counts = [len(q) for q in batch]
        assert max(counts) == kn and (kn == 1 or min(counts) < kn)


def test_crafted_fixtures_reach_every_survivor_and_fold_class(crafted):
    classes = {q: query_classes(_q(crafted, q)) for b in CRAFTED_BATCHES.values() for q in b}
    surv = [k["survivors"] for cl in classes.values() for k in cl]
    for top_n in TOP_NS:
        assert min(surv) < top_n and top_n in surv and max(surv) > top_n, top_n
    assert CHUNK in surv and any(top_n < s_ <= 32 for s_ in surv for top_n in TOP_NS)  # the CTA's sort from 32 to 1024 entries
    # several folds of fused_topn_kernel: more than one and more than two tiles of candidates
    cand = candidates(classes[("A", "B")], MAX_TOPN)
    assert cand > 2 * TOPN_TILE, cand
    assert any(TOPN_TILE < candidates(cl, t) for cl in classes.values() for t in (100, 127))


def test_extreme_docids_make_the_last_window_bound_overflow_free():
    ex = _extreme()
    X = ex["X"].ids
    assert X[0] == 1 and X[-1] == 0xFFFFFFFE and ex["Y"].ids[-1] == 0xFFFFFFFE and ex["Z"].ids[0] == 1
    assert int(X[-1]) + 1 == 0xFFFFFFFF and n_chunks(len(X)) >= 2  # k_hi of the last chunk
    assert query_classes(_q(ex, ("X", "Y", "Z")))[-1]["survivors"] > 0


def test_mask_filtered_fixtures_drive_with_a_list_that_is_not_the_shortest(masked):
    terms = masked
    for q in MASK_QUERIES:
        t = _q(terms, q)
        order = aggregate_order(t)
        by_len = sorted(range(len(t)), key=lambda i: len(t[i].ids))
        assert order != by_len and len(t[order[0]].ids) > min(len(x.ids) for x in t), q
        assert driver_chunks(t) > old_sizing_items(t), q
    # the batch of 200 outgrows every slack of a scratch sized from the shortest lists (FusedScratch::need)
    batch = [MASK_QUERIES[i % 3] for i in range(200)]
    old = sum(old_sizing_items(_q(terms, q)) for q in batch)
    new = sum(driver_chunks(_q(terms, q)) for q in batch)
    assert new > old + old // 4 + 1024 and new * MAX_TOPN > old * MAX_TOPN + old * MAX_TOPN // 4 + 4096, (old, new)


def test_the_three_child_mask_shape_sums_in_an_order_that_matters(masked):
    """With two children the sum commutes; with three the aggregate order decides the score bits of some hits."""
    terms = masked
    t = _q(terms, MASK_QUERIES[1])
    order = aggregate_order(t)
    by_len = sorted(range(len(t)), key=lambda i: len(t[i].ids))
    assert len(t) == 3 and order != by_len
    docs = reduce(np.intersect1d, [x.ids for x in t])
    pos = [np.searchsorted(x.ids, docs) for x in t]
    P = ol.postings()
    idf = [P.orc_idf_bm25(N_DOCS, x.estimated) for x in t]
    differ = 0
    for i in range(len(docs)):
        def score(o):
            return ol.oracle_score(ol.SCORER_BM25STD, [int(t[c].freqs[pos[c][i]]) for c in o], [1.0] * 3, [idf[c] for c in o],
                                   [WEIGHTS[c] for c in o], AGG_WEIGHT, 100 + i % 400, 1, 1.0, N_DOCS, 250.0, 2)
        differ += np.float64(score(order)).tobytes() != np.float64(score(by_len)).tobytes()
    assert len(docs) > 500 and differ > 0, (len(docs), differ)


def test_the_candidate_split_fixture_needs_two_launches():
    per_query = n_chunks(1_000_000)
    assert per_query == 977 and 900 * per_query > MAX_CAND // MAX_TOPN == 786_432
    assert launch_split([per_query] * 900, MAX_TOPN) == 2 and launch_split([per_query] * 900, 10) == 1


# ------------------------------------------------------------------------------------------------
# GPU: the fused batch against the oracle
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ps():
    from redisearch_b200 import postings

    return postings


@pytest.fixture(scope="module")
def doc_table():
    rng = np.random.default_rng(9)
    doc_len = rng.integers(1, 900, N_DOCS + 1).astype(np.uint32)
    doc_score = rng.choice(np.array([1.0, 0.5, 0.75, 0.25, 0.9], dtype=np.float32), N_DOCS + 1)
    max_freq = rng.integers(1, 60, N_DOCS + 1).astype(np.uint32)
    return {"doc_len": doc_len, "doc_score": doc_score, "max_freq": max_freq, "avg": float(doc_len[1:].mean())}


class Oracle:
    """Expected replies: docIds from numpy's intersection, each hit scored by the oracle with the freqs in aggregate order"""

    def __init__(self, table):
        self.t, self.cache = table, {}

    def full(self, terms, scorer):
        key = (tuple(x.name for x in terms), scorer, id(self.t))
        if key not in self.cache:
            order = aggregate_order(terms)
            docs = reduce(np.intersect1d, [x.ids for x in terms])
            pos = [np.searchsorted(x.ids, docs) for x in terms]
            t = self.t
            args = [[terms[c].params[1] for c in order], [terms[c].params[2] for c in order], [terms[c].params[0] for c in order]]
            slop = max(1, len(terms) - 1)
            avg = t["avg"] if t else 250.0
            sc = np.empty(len(docs), dtype=np.float64)
            for i, d in enumerate(docs.tolist()):
                fr = [int(terms[c].freqs[pos[c][i]]) for c in order]
                if t:
                    dl, mf, ds = int(t["doc_len"][d]), int(t["max_freq"][d]), float(t["doc_score"][d])
                else:
                    dl, mf, ds = 0, 1, 1.0  # no doc table: the kernels read 0 / 1 / 1.0
                sc[i] = ol.oracle_score(scorer, fr, *args, agg_weight(scorer), dl, mf, ds, N_DOCS, avg, slop)
            rank = np.lexsort((docs, -sc))
            self.cache[key] = (docs[rank], sc[rank])
        return self.cache[key]


def _assert_tanh_ranking_is_determined(scores):
    u = np.unique(scores)
    gaps = np.diff(u)
    assert not (gaps <= 1e-12 * np.maximum(1.0, np.abs(u[1:]))).any(), "two TANH scores within 1e-12: the ranking is not determined"


def _check(got, exp, top_n, scorer, what):
    gi, gs, gt = got
    ei, es = exp
    k = min(top_n, len(ei))
    assert gt == len(ei), (what, top_n, gt, len(ei))
    assert gi.tolist() == ei[:k].tolist(), (what, top_n)
    if scorer == ol.SCORER_BM25STD_TANH:
        _assert_tanh_ranking_is_determined(es)
        assert (np.abs(gs - es[:k]) <= 1e-12 * np.maximum(1.0, np.abs(es[:k]))).all(), (what, top_n)
    else:
        assert gs.tobytes() == es[:k].tobytes(), (what, top_n, gs[:4], es[:4])


def _run_fused(ps, queries, top_n, scorer, table, expected_launches):
    """one II_SearchTopNBatch; asserts it ran as `expected_launches` fused launches of four kernels each"""
    batch = ps.SearchBatch([([x.pl for x in q], [x.params for x in q]) for q in queries], top_n)
    ps.stats(reset=True)
    got = batch.run(False, scorer, agg_weight(scorer), N_DOCS, table["avg"] if table else 250.0, table["dt"] if table else None)
    launches = ps.stats().kernel_launches
    assert launches == 4 * expected_launches, f"{launches} kernel launches: the batch did not run fused ({expected_launches} launches of 4)"
    return got


def _attach(ps, terms):
    """upload every Term once (pl) and give it (weight, idf, bm25_idf) in its query-independent form; a Term with raw
    postings is written as IndexBlocks and read back through its field-mask filter"""
    P = ol.postings()
    for k, (name, t) in enumerate(sorted(terms.items())):
        if getattr(t, "pl", None) is not None:
            pass
        elif hasattr(t, "raw"):
            raw, fr, keep = t.raw
            codec, flt, dropped = MASK_CODEC[name]
            ix = ol.InvIndex(codec)
            for d, f, kp in zip(raw.tolist(), fr.tolist(), keep.tolist()):
                ix.add(d, f, (flt | 1) if kp else dropped)
            t.pl = ps.PostingList.from_blocks(ix.blocks(), codec, field_mask_filter=flt)
            assert len(t.pl) == len(t.ids) and t.pl.num_estimated() == t.estimated == len(raw), name  # the estimate stays unfiltered
            got, _, gf = ps.union([t.pl]).fetch()
            assert got.tolist() == t.ids.tolist() and gf[0].tolist() == t.freqs.tolist(), name
        else:
            t.pl = ps.PostingList.from_arrays(t.ids.astype(np.uint64), t.freqs)
        t.params = (WEIGHTS[k % len(WEIGHTS)], P.orc_idf(N_DOCS, t.estimated), P.orc_idf_bm25(N_DOCS, t.estimated))


@pytest.fixture(scope="module")
def gpu_crafted(ps, crafted, doc_table):
    _attach(ps, crafted)
    t = dict(doc_table)
    t["dt"] = ps.DocTable(N_DOCS, t["doc_len"], t["doc_score"], t["max_freq"])
    return crafted, t


def _chain_sample(ps, queries, got, top_n, scorer, table):
    """the per-query chain (II_SearchTopN) gives the same rows"""
    for q, (gi, gs, gt) in list(zip(queries, got))[::3]:
        ei, es, et = ps.search_topn([x.pl for x in q], False, scorer, [x.params for x in q], agg_weight(scorer), N_DOCS,
                                    table["avg"] if table else 250.0, table["dt"] if table else None, top_n)
        assert et == gt and ei.tolist() == gi.tolist() and es.tobytes() == gs.tobytes(), [x.name for x in q]


@pytest.mark.gpu
@pytest.mark.parametrize("scorer", range(7))
def test_membership_paths_and_chunk_classes_equal_the_oracle(ps, gpu_crafted, scorer):
    """all-fit / list-by-list / pivot paths and their edges, every instantiation kN, driver lengths 1..1025, per-chunk
    survivors around top_n and several folds of the per-query top-N, at top_n 1 / 7 / 10 / 100 / 127 / 128"""
    corpus, table = gpu_crafted
    orc = Oracle(table)
    for kn, names in CRAFTED_BATCHES.items():
        queries = [_q(corpus, q) for q in names]
        for top_n in TOP_NS:
            got = _run_fused(ps, queries, top_n, scorer, table, 1)
            for q, g in zip(queries, got):
                _check(g, orc.full(q, scorer), top_n, scorer, (kn, [x.name for x in q]))
            if top_n in (7, 128):
                _chain_sample(ps, queries, got, top_n, scorer, table)


@pytest.mark.gpu
def test_equal_keys_across_folds_are_ranked_by_docid(ps, gpu_crafted):
    """DOCSCORE with two doc scores: thousands of equal keys reach fused_topn_kernel, and after each fold its threshold
    must still let an equal key with a smaller docId in"""
    corpus, table = gpu_crafted
    rng = np.random.default_rng(4)
    t = dict(table)
    t["doc_score"] = rng.choice(np.array([1.0, 0.5], dtype=np.float32), N_DOCS + 1)
    t["dt"] = ps.DocTable(N_DOCS, t["doc_len"], t["doc_score"], t["max_freq"])
    orc = Oracle(t)
    queries = [_q(corpus, ("A", "B")), _q(corpus, ("A", "C", "B"))]
    assert candidates(query_classes(queries[0]), MAX_TOPN) > 2 * TOPN_TILE
    for top_n in TOP_NS:
        got = _run_fused(ps, queries, top_n, ol.SCORER_DOCSCORE, t, 1)
        for q, g in zip(queries, got):
            _check(g, orc.full(q, ol.SCORER_DOCSCORE), top_n, ol.SCORER_DOCSCORE, [x.name for x in q])
        _chain_sample(ps, queries, got, top_n, ol.SCORER_DOCSCORE, t)


@pytest.mark.gpu
@pytest.mark.parametrize("scorer", range(7))
def test_docids_1_and_0xfffffffe_without_a_doc_table(ps, scorer):
    ex = _extreme()
    _attach(ps, ex)
    orc = Oracle(None)
    queries = [_q(ex, q) for q in EXTREME_QUERIES]
    for top_n in (1, 10, 128):
        got = _run_fused(ps, queries, top_n, scorer, None, 1)
        for q, g in zip(queries, got):
            _check(g, orc.full(q, scorer), top_n, scorer, [x.name for x in q])
        _chain_sample(ps, queries, got, top_n, scorer, None)


@pytest.fixture(scope="module")
def gpu_masked(ps, masked, doc_table):
    _attach(ps, masked)
    t = dict(doc_table)
    t["dt"] = ps.DocTable(N_DOCS, t["doc_len"], t["doc_score"], t["max_freq"])
    return masked, t


@pytest.mark.gpu
def test_a_batch_of_mask_filtered_queries_outgrowing_the_scratch_runs_fused(ps, gpu_masked):
    """200 queries whose driver (the first list by estimate) is longer than their shortest child: the work items, the scratch
    and the candidate budget come from the driver.  Sized from the shortest child, this batch outgrows every slack of the
    grow-only scratch (the batch scratch only grows within a process, so this runs before the larger batches below)."""
    terms, table = gpu_masked
    orc = Oracle(table)
    queries = [_q(terms, MASK_QUERIES[i % 3]) for i in range(200)]
    got = _run_fused(ps, queries, MAX_TOPN, ol.SCORER_BM25STD, table, 1)
    for q, g in zip(queries, got):
        _check(g, orc.full(q, ol.SCORER_BM25STD), MAX_TOPN, ol.SCORER_BM25STD, [x.name for x in q])
    _chain_sample(ps, queries[:6], got[:6], MAX_TOPN, ol.SCORER_BM25STD, table)


@pytest.mark.gpu
@pytest.mark.parametrize("scorer", range(7))
def test_mask_filtered_children_keep_the_aggregate_order(ps, gpu_masked, scorer):
    """the 2-child shape (an unfiltered term AND a filtered one with more raw and fewer kept postings) and the 3-child shape
    whose score bits depend on the aggregate order, each alone in a batch"""
    terms, table = gpu_masked
    orc = Oracle(table)
    for names in MASK_QUERIES:
        q = _q(terms, names)
        for top_n in (1, 10, 128):
            got = _run_fused(ps, [q], top_n, scorer, table, 1)
            _check(got[0], orc.full(q, scorer), top_n, scorer, names)
            _chain_sample(ps, [q], got, top_n, scorer, table)


@pytest.mark.gpu
def test_a_batch_past_the_candidate_budget_splits_into_two_launches(ps, doc_table):
    """900 queries x 977 driver chunks x top_n 128 > kMaxCand slots: two launches, every repeat equal to the oracle"""
    rng = np.random.default_rng(12)
    perm = rng.permutation(np.arange(1, N_DOCS + 1, dtype=np.int64))
    M, S = 1_000_000, 5_000
    lists = {"P": perm[:M], "Q": perm[M - S:2 * M - S], "R": np.concatenate([perm[2 * M - 2 * S:3 * M - 3 * S], perm[:S]])}
    terms = {k: Term(k, np.sort(v), stepped_freqs(rng, M)) for k, v in lists.items()}
    _attach(ps, terms)
    table = dict(doc_table)
    table["dt"] = ps.DocTable(N_DOCS, table["doc_len"], table["doc_score"], table["max_freq"])
    distinct = [("P", "Q"), ("Q", "R"), ("R", "P")]
    queries = [_q(terms, distinct[i % 3]) for i in range(900)]
    assert all(driver_chunks(q) == 977 for q in queries[:3])
    assert launch_split([977] * 900, MAX_TOPN) == 2
    got = _run_fused(ps, queries, MAX_TOPN, ol.SCORER_BM25STD, table, 2)
    orc = Oracle(table)
    for i, (q, g) in enumerate(zip(queries, got)):
        exp = orc.full(q, ol.SCORER_BM25STD)
        assert len(exp[0]) == S
        _check(g, exp, MAX_TOPN, ol.SCORER_BM25STD, (i, distinct[i % 3]))
    _chain_sample(ps, queries[:3], got[:3], MAX_TOPN, ol.SCORER_BM25STD, table)
