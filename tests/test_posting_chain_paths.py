"""The per-query posting-list chain (II_IntersectEx / II_IntersectPhrase / II_Union / II_Score / II_ResultSet_TopN, and
II_SearchTopN[Batch] off the fused route) held to the oracle at the branch edges of its kernels: intersect_kernel (and_probe),
scan_kernel, gather_kernel, score_kernel, topn_kernel, the union's mark / popc / expand / fill_freq, mask_flags / mask_compact,
numeric_flags / numeric_compact, phrase_filter + flag_compact, min_offset_delta_kernel and merge_write_kernel.

The CPU half restates what the host and the kernels decide (the aggregate child order, the driver and the kernel list order,
the probe window of every driver chunk and list, staged or not, the early exit, the scan rounds, the union bitmap words and
32-word blocks, the compaction chunks), pins the constants those decisions rest on to the sources, shows that the fixtures
reach every class, and shows that the expected-answer checks reject a dropped hit, a swapped freq row and a score one ulp off.

The GPU half runs the fixtures through the chain and compares with exact host answers: docIds from numpy set algebra or the
oracle's run_intersect, freq rows from the lists at their aggregate-order row, scores from oracle/scorer_oracle.c (GetSlop from
ol.min_offset_delta, phrase membership from ol.within_range), BM25STD.TANH within 1e-12.  Every call checks the kernel launch
count of the chain, so a silent move to the fused route (or to any other route) fails the test.
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
MAX_LISTS, PHRASE_MAX_LISTS, UNION_FLAT_MAX = 32, 8, 20
TOPN_DEVICE_MAX = 1024  # II_ResultSet_TopN: a larger k is partial-sorted on the host
TOPN_WARPS = 8          # topn_kernel: 256 threads, one list per warp
COMPACT_CHUNK = 1024    # mask_flags / numeric_flags / flag_count: one CTA per 1,024 entries
SCAN_ROUND = 1024       # scan_kernel: one CTA of 1,024 threads, a carry between rounds

# kernel launches the chain counts in II_Stats (ii_host.cpp): intersect + scan + gather; the phrase filter adds phrase_filter,
# flag_count, scan and flag_compact; II_SearchTopN adds the scorer and topn_kernel (the fused route counts 4 per batch)
L_AND, L_PHRASE, L_SCORE, L_SLOP, L_TOPN, L_SEARCH, L_FILTER = 3, 7, 1, 1, 1, 5, 3


def union_launches(n):
    """union_enqueue counts mark and fill_freq per child (empty ones included) plus popc, scan and expand"""
    return 3 + 2 * n


N_DOCS = 3_000_000
AGG = 0.7
WEIGHTS = (1.0, 0.5, 1.5, 0.3, 1.25, 0.75, 1.1, 0.9)
ALL_SCORERS = tuple(range(7))
LEGACY = (ol.SCORER_BM25, ol.SCORER_TFIDF, ol.SCORER_TFIDF_DOCNORM)


def agg_weight(scorer):
    """BM25STD.TANH at 0.1: its scores stay clear of tanh's saturation, where distinct scores crowd within 1e-12"""
    return 0.1 if scorer == ol.SCORER_BM25STD_TANH else AGG


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(r"\b" + name + r"\s*=\s*(\d+)\s*[;,]", text)
    assert m, name
    return int(m.group(1))


def test_constants_match_the_sources():
    h, cu, host = _read("ii_kernels.h"), _read("ii_kernels.cu"), _read("ii_host.cpp")
    assert _const(h, "kIIThreads") == II_THREADS and _const(h, "kIIItems") == II_ITEMS
    assert re.search(r"\bkIIChunk\s*=\s*kIIThreads\s*\*\s*kIIItems\s*;", h) and II_THREADS * II_ITEMS == CHUNK
    assert _const(h, "kIISmemElems") == SMEM_ELEMS
    assert _const(h, "kIIMaxLists") == MAX_LISTS and _const(h, "kPhraseMaxLists") == PHRASE_MAX_LISTS
    assert _const(h, "kIIUnionFlatMax") == UNION_FLAT_MAX
    # and_probe stages a window of at most kIISmemElems entries, its end is the lower bound of a_hi + 1
    probe = cu[cu.index("void and_probe("):cu.index("cta_survivor_rank(")]
    assert re.search(r"staged\s*=\s*range\s*<=\s*\(uint32_t\)kIISmemElems", probe)
    assert "a_hi + 1u" in probe and "__syncthreads_or(any)" in probe
    # scan_kernel: one CTA, rounds of 1,024 counts with a carry
    scan = cu[cu.index("scan_kernel("):cu.index("// scorers")]
    assert "base += 1024" in scan and "s_carry" in scan
    assert re.search(r"scan_kernel<<<1,\s*1024", cu)
    # the compaction chunk of the mask / numeric / phrase filters
    for k in ("mask_flags_kernel", "numeric_flags_kernel", "flag_count_kernel", "mask_compact_kernel", "numeric_compact_kernel"):
        body = cu[cu.index(k + "("):]
        body = body[:body.index("\n}\n")]
        assert "blockIdx.x * 1024u" in body, k
    assert cu.count("(n + 1023) / 1024") >= 2 and "(cap_len + 1023) / 1024" in cu
    # topn_kernel: 8 warps' lists per CTA; II_ResultSet_TopN: k above 1,024 on the host
    topn = cu[cu.index("topn_kernel("):]
    assert "blockIdx.x * 8 + warp" in topn[:topn.index("\n}\n")]
    assert re.search(r"topn_kernel<<<grid,\s*256,", cu)
    assert re.search(r"ii_topn_lists\(uint32_t m\) \{ return grid_for\(m, 256, 132 \* 2\) \* 8; \}", cu)  # topn_lists below
    tn = host[host.index("size_t II_ResultSet_TopN("):]
    assert re.search(r"if \(k > (\d+)\)", tn).group(1) == str(TOPN_DEVICE_MAX)
    # the union bitmap spans docIds 0 .. max_id
    assert "nwords = plan.max_id / 32 + 1" in host


# ------------------------------------------------------------------------------------------------
# the host's and the kernels' decisions, restated
# ------------------------------------------------------------------------------------------------
class Term:
    """One child: its docIds and freqs after any field-mask filter, and num_estimated (the unfiltered count)."""

    def __init__(self, name, ids, freqs, estimated=None):
        self.name, self.ids, self.freqs = name, np.asarray(ids, dtype=np.int64), np.asarray(freqs, dtype=np.uint32)
        self.estimated = len(self.ids) if estimated is None else estimated


def aggregate_order(terms, modes, in_order=False):
    """intersect_enqueue: a stable sort by num_estimated (intersection.rs:110-145), NOT / OPTIONAL children behind every
    required one in their given order (and_sort_key: 2^62); an in-order phrase keeps the given order"""
    if in_order:
        return list(range(len(terms)))
    return sorted(range(len(terms)), key=lambda i: float(terms[i].estimated) if modes[i] == 0 else 2.0 ** 62)


def kernel_order(terms, modes, order):
    """intersect_enqueue: the driver is the REQUIRED child with the fewest actual entries (first in aggregate order on a tie);
    the other lists follow ascending by length, stable in aggregate order.  Returns aggregate slots in kernel order."""
    drv = None
    for j, c in enumerate(order):
        if modes[c] == 0 and (drv is None or len(terms[c].ids) < len(terms[order[drv]].ids)):
            drv = j
    rest = sorted([j for j in range(len(order)) if j != drv], key=lambda j: len(terms[order[j]].ids))
    return [drv] + rest


def n_chunks(n):
    return (n + CHUNK - 1) // CHUNK


def probe_classes(terms, modes):
    """intersect_kernel / and_probe, per driver chunk: the window [lower_bound(A[start]), lower_bound(A[end-1] + 1)) of every
    probed list, whether it is staged (<= kIISmemElems entries), the early exit (no entry alive: later lists are not probed),
    where driver entries sit against a window, and the chunk's survivors"""
    order = aggregate_order(terms, modes)
    ko = kernel_order(terms, modes, order)
    A = terms[order[ko[0]]].ids
    out = []
    for c in range(n_chunks(len(A))):
        doc = A[c * CHUNK:(c + 1) * CHUNK]
        lo_key, hi_key = int(doc[0]), int(doc[-1]) + 1
        alive = np.ones(len(doc), dtype=bool)
        k = {"windows": [], "staged": [], "early_exit": False, "edges": set(), "modes": []}
        for j in ko[1:]:
            if not alive.any():
                k["early_exit"] = True
                break
            B, mode = terms[order[j]].ids, modes[order[j]]
            lo, hi = int(np.searchsorted(B, lo_key, "left")), int(np.searchsorted(B, hi_key, "left"))
            k["windows"].append(hi - lo)
            k["staged"].append(hi - lo <= SMEM_ELEMS)
            k["modes"].append(mode)
            if hi > lo:
                W = B[lo:hi]
                d = doc[alive]
                for name, hit in (("first", d == W[0]), ("last", d == W[-1]), ("below", d < W[0]), ("above", d > W[-1])):
                    if hit.any():
                        k["edges"].add((mode, name))
                if mode and (doc[0] == W[0] or doc[-1] == W[-1]):
                    k["edges"].add((mode, "chunk_edge_member"))
            found = np.isin(doc, B)
            if mode == 0:
                alive &= found
            elif mode == 1:
                alive &= ~found
        k["survivors"] = int(alive.sum())
        out.append(k)
    return out


def and_expected(terms, modes, in_order=False):
    """docIds by numpy set algebra, the aggregate child order and the freq rows at their aggregate slot (NOT children and
    absent OPTIONAL children are virtual results: freq 0)"""
    order = aggregate_order(terms, modes, in_order)
    docs = reduce(np.intersect1d, [t.ids for t, m in zip(terms, modes) if m == 0])
    for t, m in zip(terms, modes):
        if m == 1:
            docs = np.setdiff1d(docs, t.ids)
    return docs, order, freq_rows(terms, order, modes, docs)


def freq_rows(terms, order, modes, docs):
    rows = np.zeros((len(order), len(docs)), dtype=np.uint32)
    for j, c in enumerate(order):
        if modes[c] == 1 or not len(docs) or not len(terms[c].ids):
            continue
        p = np.minimum(np.searchsorted(terms[c].ids, docs), len(terms[c].ids) - 1)
        hit = terms[c].ids[p] == docs
        rows[j, hit] = terms[c].freqs[p[hit]]
    return rows


def check_set(got, exp, what):
    """got = (docIds, freq rows [aggregate slot][hit], child order); exp = (docIds, child order, freq rows)"""
    gi, gf, go = got
    ei, eo, ef = exp
    assert len(gi) == len(ei) and np.array_equal(np.asarray(gi, dtype=np.int64), np.asarray(ei, dtype=np.int64)), (what, len(gi), len(ei))
    assert list(go) == list(eo), (what, list(go), list(eo))
    assert gf.shape == ef.shape and np.array_equal(gf, ef), (what, "freq rows")


def check_scores(got, exp, scorer, what):
    """bits equal; BM25STD.TANH within 1e-12 (libm vs device tanh)"""
    got, exp = np.asarray(got, dtype=np.float64), np.asarray(exp, dtype=np.float64)
    assert got.shape == exp.shape, what
    if scorer == ol.SCORER_BM25STD_TANH:
        bad = np.abs(got - exp) > 1e-12 * np.maximum(1.0, np.abs(exp))
    else:
        bad = got.view(np.uint64) != exp.view(np.uint64)
    assert not bad.any(), (what, scorer, int(bad.sum()), got[bad][:3], exp[bad][:3])


def check_ranking(got_ids, got_scores, docs, scores, k, what):
    """the top k by (score desc, docId asc), the scores' bits equal"""
    rank = np.lexsort((docs, -scores))[:k]
    assert np.asarray(got_ids, dtype=np.int64).tolist() == docs[rank].tolist(), (what, k)
    assert np.asarray(got_scores, dtype=np.float64).tobytes() == scores[rank].tobytes(), (what, k)


def sample(m, limit=12_000, extra=()):
    """every hit when there are few, else ~1,500 spread over the set plus both ends and the given indices"""
    if m <= limit:
        return np.arange(m)
    idx = set(range(0, m, max(1, m // 1500))) | set(range(60)) | set(range(m - 60, m))
    idx |= {i for e in extra for i in range(e - 3, e + 3) if 0 <= i < m}
    return np.array(sorted(idx))


class Table:
    """doc_len / max_freq / doc_score by docId (None: no doc table, the kernels read 0 / 1 / 1.0)"""

    def __init__(self, rng=None, two_scores=False):
        if rng is None:
            self.doc_len = self.doc_score = self.max_freq = None
            self.avg = 250.0
            return
        self.doc_len = rng.integers(1, 900, N_DOCS + 1).astype(np.uint32)
        vals = [1.0, 0.5] if two_scores else [1.0, 0.5, 0.75, 0.25, 0.9]
        self.doc_score = rng.choice(np.array(vals, dtype=np.float32), N_DOCS + 1)
        self.max_freq = rng.integers(1, 60, N_DOCS + 1).astype(np.uint32)
        self.avg = float(self.doc_len[1:].mean())

    def of(self, d):
        if self.doc_len is None:
            return 0, 1, 1.0
        return int(self.doc_len[d]), int(self.max_freq[d]), float(self.doc_score[d])


def params_of(terms):
    P = ol.postings()
    return [(WEIGHTS[k % len(WEIGHTS)], P.orc_idf(N_DOCS, t.estimated), P.orc_idf_bm25(N_DOCS, t.estimated)) for k, t in enumerate(terms)]


def expected_scores(scorer, docs, rows, orders, params, table, idx, slop):
    """oracle_score of hits idx: the present children (freq != 0) of each hit in its aggregate order.  orders: one order for
    every hit, or a callable hit -> order; slop: an int or a callable hit -> GetSlop"""
    out = np.empty(len(idx), dtype=np.float64)
    for n, i in enumerate(idx.tolist()):
        order = orders(i) if callable(orders) else orders
        fr = [(c, int(f)) for c, f in zip(order, rows(i) if callable(rows) else rows[:, i]) if f]
        dl, mf, ds = table.of(int(docs[i]))
        out[n] = ol.oracle_score(scorer, [f for _, f in fr], [params[c][1] for c, _ in fr], [params[c][2] for c, _ in fr],
                                 [params[c][0] for c, _ in fr], agg_weight(scorer), dl, mf, ds, N_DOCS, table.avg,
                                 slop(i) if callable(slop) else slop)
    return out


# ------------------------------------------------------------------------------------------------
# fixtures (numpy only: the CPU tests show what they reach, the GPU tests run them)
# ------------------------------------------------------------------------------------------------
def stepped_freqs(rng, n, top=29):
    """freqs in 1..top whose neighbours always differ: a row off by one changes the answer"""
    return (1 + np.cumsum(rng.integers(1, top, n)) % top).astype(np.uint32)


NB = 1_200_000


def _probe():
    """B = the even docIds up to 2.4M; A = a driver laid out chunk by chunk against B.  N (NOT, multiples of 3) and O
    (OPTIONAL, multiples of 5) are longer than B, so the kernel probes B first; O_none (odd docIds) never matches a hit and
    O_all (B's docIds) matches every one; E is empty."""
    rng = np.random.default_rng(2026)
    B = 2 * np.arange(1, NB + 1, dtype=np.int64)
    chunks, s = [], 10

    def edges_chunk(W):
        # a window of exactly W entries of B: A[0] = B[s] - 1 below it, A[1] = its first entry, A[-2] its last, A[-1] above it
        nonlocal s
        first, last = B[s], B[s + W - 1]
        inner = rng.choice(B[s + 1:s + W - 1], 500, replace=False)
        odd = rng.choice(B[s + 1:s + W - 2] + 1, 1020 - 500, replace=False)
        chunks.append(np.sort(np.concatenate([[first - 1, first, last, last + 1], inner, odd])))
        s += W + 1

    def count_chunk(W, m, n=CHUNK):
        # n entries of which exactly m are in B
        nonlocal s
        mem = B[s:s + W] if m == W else rng.choice(B[s:s + W], m, replace=False)
        odd = rng.choice(B[s:s + W] + 1, n - m, replace=False)
        chunks.append(np.sort(np.concatenate([mem, odd])))
        s += W + 1

    def none_chunk(W):
        # no entry in B: the CTA leaves and_probe after B, before the NOT / OPTIONAL lists
        nonlocal s
        chunks.append(np.sort(rng.choice(B[s:s + W] + 1, CHUNK, replace=False)))
        s += W + 1

    def member_edge_chunk(first_mod, last_mod, W=3000):
        # every entry in B; the chunk's first entry in the list of first_mod, its last in that of last_mod: the NOT / OPTIONAL
        # windows begin or end on a driver entry
        nonlocal s
        v = B[s:s + W]
        lo = v[v % first_mod == 0][0]
        hi = v[v % last_mod == 0][-1]
        mid = v[(v > lo) & (v < hi)]
        chunks.append(np.sort(np.concatenate([[lo, hi], rng.choice(mid, CHUNK - 2, replace=False)])))
        s += W + 1

    count_chunk(3000, 700)
    edges_chunk(SMEM_ELEMS - 1)
    edges_chunk(SMEM_ELEMS)
    edges_chunk(SMEM_ELEMS + 1)
    count_chunk(CHUNK, CHUNK)        # full
    count_chunk(3000, 0)             # zero survivors between full chunks
    count_chunk(CHUNK, CHUNK)
    count_chunk(3000, 400)
    none_chunk(3000)                 # the early exit, survivors on both sides
    count_chunk(3000, 300)
    member_edge_chunk(6, 10)         # NOT window starts on the chunk's first entry, OPTIONAL window ends on its last
    member_edge_chunk(10, 6)
    count_chunk(3000, 1)
    edges_chunk(1_050_000)           # a window over 1M entries
    count_chunk(2000, 150, n=300)    # partial last chunk
    assert s <= NB
    A = np.concatenate(chunks)
    assert (np.diff(A) > 0).all()
    ids = {"A": A, "B": B, "N": 3 * np.arange(1, 1_300_001, dtype=np.int64), "O": 5 * np.arange(1, 1_400_001, dtype=np.int64),
           "O_none": 2 * np.arange(0, NB + 50_000, dtype=np.int64) + 1, "O_all": B.copy(), "E": np.zeros(0, dtype=np.int64)}
    return {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


PROBE_QUERIES = [  # (names, modes)
    (("A", "B"), (0, 0)),
    (("A", "B", "N", "O"), (0, 0, 1, 2)),
    (("N", "B", "A", "O"), (1, 0, 0, 2)),
    (("A", "B", "E"), (0, 0, 1)),
    (("A", "O_none", "B"), (0, 2, 0)),
    (("A", "B", "O_all"), (0, 0, 2)),
]


def _wide():
    """32 lists sharing 3,000 docIds, plus a NOT and an OPTIONAL list: the 2 / 3 / 8 / 16 / 32-child ANDs"""
    rng = np.random.default_rng(88)
    shared = rng.choice(N_DOCS - 10, 3000, replace=False) + 1
    ids = {}
    for k in range(MAX_LISTS + 1):
        ids[f"W{k}"] = np.union1d(shared, rng.choice(N_DOCS - 10, 5_000 + 6_000 * k, replace=False) + 1)
    ids["WN"] = np.union1d(rng.choice(shared, 400, replace=False), rng.choice(N_DOCS - 10, 50_000, replace=False) + 1)
    ids["WO"] = np.union1d(rng.choice(shared, 1500, replace=False), rng.choice(N_DOCS - 10, 80_000, replace=False) + 1)
    return {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


def wide_query(n):
    """n children: the first n - 2 W lists required, then a NOT and an OPTIONAL child (n = 2: two required lists)"""
    if n == 2:
        return ("W0", "W1"), (0, 0)
    return tuple(f"W{k}" for k in range(n - 2)) + ("WN", "WO"), (0,) * (n - 2) + (1, 2)


WIDE_NS = (2, 3, 8, 16, 32)


def _lengths():
    """Drivers of 1, 1,023, 1,024, 1,025, 2,048 and 1,100,000 entries (1,075 chunks: scan_kernel carries across two rounds)
    against P, which holds every docId in 1..3M except those removed chunk by chunk: chunk c of the long driver D keeps all
    its entries in P (c % 4 in 0, 3), none (c % 4 == 1) or about half (c % 4 == 2)."""
    rng = np.random.default_rng(5150)
    D = np.sort(rng.choice(N_DOCS - 10, 1_100_000, replace=False) + 1)
    drop = []
    for c in range(n_chunks(len(D))):
        part = D[c * CHUNK:(c + 1) * CHUNK]
        if c % 4 == 1:
            drop.append(part)
        elif c % 4 == 2:
            drop.append(part[rng.random(len(part)) < 0.5])
    P = np.setdiff1d(np.arange(1, N_DOCS + 1, dtype=np.int64), np.concatenate(drop))
    ids = {"D": D, "P": P}
    for n in (1023, 1024, 1025, 2048):
        ids[f"L{n}"] = np.sort(rng.choice(D, n, replace=False))
    ids["L1"] = rng.choice(np.intersect1d(D, P), 1)  # a hit
    return {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


LENGTH_DRIVERS = ("L1", "L1023", "L1024", "L1025", "L2048", "D")


def _masked():
    """Field-mask-filtered children keep num_estimated = the unfiltered count: the estimate sorts them last while their
    filtered length makes them the driver.  raw = every posting written, keep = what the filter keeps."""
    rng = np.random.default_rng(31)
    U = np.sort(rng.choice(400_000, 100_000, replace=False) + 1)
    U2 = np.sort(rng.choice(400_000, 20_000, replace=False) + 1)
    U3 = np.union1d(U2[::2], rng.choice(400_000, 50_000, replace=False) + 1)
    terms = {n: Term(n, v, stepped_freqs(rng, len(v))) for n, v in (("U", U), ("U2", U2), ("U3", U3))}
    for name, raw_n, kept_from, n_kept in (("M1", 150_000, U, 2_000), ("M2", 120_000, np.intersect1d(U2, U3), 3_000)):
        kept = np.union1d(rng.choice(kept_from, min(len(kept_from), n_kept - 400), replace=False), rng.choice(400_000, 400, replace=False) + 1)
        rest = rng.permutation(np.setdiff1d(rng.choice(400_000, raw_n + 10_000, replace=False) + 1, kept))[:raw_n - len(kept)]
        raw = np.union1d(kept, rest)
        fr = stepped_freqs(rng, raw_n)
        keep = np.isin(raw, kept)
        terms[name] = Term(name, raw[keep], fr[keep], estimated=raw_n)
        terms[name].raw = (raw, fr, keep)
    return terms


# codec, field-mask filter, the mask of a posting the filter drops (M2's filter is above bit 63: FromBlocksWideMask)
MASK_CODEC = {"M1": (ol.CODEC_FREQS_FIELDS, 0b10, 0b01), "M2": (ol.CODEC_FREQS_FIELDS_WIDE, 1 << 100, 1 << 3)}
MASK_QUERIES = [("U", "M1"), ("U2", "M2", "U3"), ("M2", "U", "U3")]


def _union_edges():
    """docIds on the first and last bit of bitmap words 0 (docId 0 is not a document: bit 1), 31, 32, 1,023, 1,024 (the
    32-word blocks 0 / 1 and 31 / 32) and 32,767 / 32,768 (blocks 1,023 / 1,024: the scan's second round), spread over three
    children with overlaps, and the same with docId 0xFFFFFFFE added (a 512 MB bitmap)"""
    rng = np.random.default_rng(17)
    edge = sorted({x for w in (0, 31, 32, 1023, 1024, 32767, 32768) for x in (32 * w, 32 * w + 31)} - {0} | {1})
    kids = [[], [], []]
    for k, d in enumerate(edge):
        for c in range(3):
            if (k + c) % 3 != 2 or d == 1:
                kids[c].append(d)
    fill = [rng.choice(np.arange(2, 1_100_000), 3000, replace=False) for _ in range(3)]
    ids = {f"E{c}": np.union1d(kids[c], fill[c]) for c in range(3)}
    ids["Etop"] = np.union1d(ids["E2"], [0xFFFFFFFE, 0xFFFFFFFE - 31, 0xFFFFFFFE - 1])
    return edge, {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


def _union_exhaust():
    """Six children, densely overlapping, whose last docIds are 5,000, 5,000 (the same docId), 5,001 and 4,999 (neighbours),
    9,000, and one empty from the start: the UnionOrder epochs change at each of them"""
    rng = np.random.default_rng(23)
    last = (5000, 5000, 5001, 4999, 9000)
    ids = {}
    for c, end in enumerate(last):
        v = np.flatnonzero(rng.random(end + 1) < 0.45)
        ids[f"X{c}"] = np.union1d(v[v >= 1], [4998, 4999, end])  # the docIds around the ends are in every child that reaches them
    ids["X5"] = np.zeros(0, dtype=np.int64)
    return {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


def _union_many(n, seed):
    """n sparse children over 20,000 docIds: the oracle's hits list at most 16 children, so no docId is in more"""
    rng = np.random.default_rng(seed)
    ids = {}
    for c in range(n):
        ids[f"Y{c}"] = np.flatnonzero(rng.random(20_001) < 0.12)
        ids[f"Y{c}"] = ids[f"Y{c}"][ids[f"Y{c}"] >= 1]
    return {k: Term(k, v, stepped_freqs(rng, len(v))) for k, v in ids.items()}


def _mask_postings():
    """5 x 1,024 + 300 FreqsFields postings (one block decode, one compaction CTA per 1,024): masks for filters keeping none,
    all, or exactly one entry per chunk (at offsets 0, 1,023 and in between), plus the last entry of chunk 2 and the first of
    chunk 3 for a second filter"""
    rng = np.random.default_rng(41)
    n = 5 * COMPACT_CHUNK + 300
    ids = np.sort(rng.choice(2_000_000, n, replace=False) + 1)
    fr = stepped_freqs(rng, n)
    masks = np.full(n, 0b0001, dtype=np.int64)  # every posting: field 0 (the "all" filter)
    one = [c * COMPACT_CHUNK + off for c, off in enumerate((0, 1023, 511, 1, 1022))] + [5 * COMPACT_CHUNK + 299]
    masks[one] |= 0b0100
    pair = [3 * COMPACT_CHUNK - 1, 3 * COMPACT_CHUNK]
    masks[pair] |= 0b1000
    return ids, fr, masks, {"none": 0b10000, "all": 0b0001, "one_per_chunk": 0b0100, "straddle": 0b1000}


def _numeric_records():
    """Numeric records with multi-value documents whose adjacent records straddle every 1,024 boundary of the decoded array:
    the first in-range record on the left of it, on the right, or both; values at +-inf, -0.0 and 0.0"""
    rng = np.random.default_rng(99)
    n = 4 * COMPACT_CHUNK + 100
    vals = rng.choice(np.array([-np.inf, np.inf, -0.0, 0.0, 1.0, -1.0, 2.5, -7.25, 1e300, -1e-300]), n)
    step = rng.integers(1, 3, n)
    for b in range(1, 5):
        i = b * COMPACT_CHUNK
        if i < n:
            step[i] = 0  # records i - 1 and i belong to one document
    step[0] = 1
    ids = np.cumsum(step).astype(np.int64)
    # boundary 1: the left record in (0, inf), the right not; 2: the right only; 3: both; 4: three records -0.0, 0.0, inf
    vals[1023], vals[1024] = 1.0, -7.25
    vals[2047], vals[2048] = -1.0, 2.5
    vals[3071], vals[3072] = 1.0, 2.5
    vals[4095], vals[4096] = -0.0, 0.0
    ids[4097] = ids[4096]
    ids[4098:] = ids[4098:] - ids[4098] + ids[4096] + 1 + np.arange(n - 4098)
    vals[4097] = np.inf
    return ids, vals


def decoded_numeric(ids, vals):
    """the values the oracle's decoder reads back from the IndexBlocks of these records (-0.0 is stored as the integer 0)"""
    out = []
    for _, _, cnt, data in ol.numeric_blocks(ids.tolist(), vals.tolist()):
        at = 0
        for _ in range(cnt):
            used, _, v = ol.numeric_decode(data[at:])
            at += used
            out.append(v)
    return np.array(out, dtype=np.float64)


NUMERIC_RANGES = [(-np.inf, np.inf, True, True), (-np.inf, np.inf, False, False), (0.0, np.inf, False, True), (0.0, np.inf, True, False),
                  (-0.0, 0.0, True, True), (-0.0, 0.0, False, True), (-np.inf, -0.0, True, False), (np.inf, np.inf, True, True),
                  (-1.0, 1.0, False, False)]


def expected_numeric(ids, vals, lo, hi, li, hi_i):
    """the first in-range record of every document (numeric_keep: an earlier in-range record of the same docId wins)"""
    P = ol.postings()
    seen, out = set(), []
    for d, v in zip(ids.tolist(), vals.tolist()):
        if d not in seen and P.orc_numeric_in_range(v, lo, hi, int(li), int(hi_i)):
            seen.add(d)
            out.append(d)
    return np.array(out, dtype=np.int64)


def varint_len(v):
    """bytes of one RS varint (7-bit groups, +1 per continuation)"""
    return len(ol.varint_deltas([v]))


def _phrase():
    """8 Full-codec terms over 6,000 documents with crafted term positions: 1- to 5-byte varint deltas (positions up to
    300,000,000 + small, above 2^28), position 0, zero deltas (a position repeated), the same position in several terms (the
    negative-span case), spans of exactly s and s + 1 for s in 0, 1, 3, and records with no positions inside a hit."""
    rng = np.random.default_rng(4242)
    n_docs, n_terms = 6000, PHRASE_MAX_LISTS
    dens = (0.9, 0.8, 0.85, 0.75, 0.9, 0.8, 0.85, 0.9)
    pos = [dict() for _ in range(n_terms)]
    for d in range(1, n_docs + 1):
        kind = d % 6
        base = {0: 0, 1: 0, 2: 200, 3: 20_000, 4: 3_000_000, 5: 300_000_000}[kind]
        gaps = rng.integers(0, 3, n_terms) if kind != 1 else np.zeros(n_terms, dtype=np.int64)
        start = base + (0 if kind in (0, 1) else int(rng.integers(0, 50)))
        at = start + np.concatenate([[0], np.cumsum(1 + gaps[1:])])  # in-order, term t at at[t]
        for t in range(n_terms):
            if rng.random() > dens[t]:
                continue
            p = [int(at[t])]
            r = rng.random()
            if r < 0.3:
                p.append(int(at[t]) + int(rng.integers(3, 40)))
            elif r < 0.4:
                p.append(int(at[t]))  # a zero delta
            elif r < 0.5 and t:
                p.append(int(at[t - 1]))  # the previous term's position: the same position in two terms
            elif r < 0.55 and kind == 0:
                p = [0]
            if rng.random() < 0.04:
                p = []  # a record without positions
            pos[t][d] = sorted(p)
    return pos


def _phrase_terms(pos):
    rng = np.random.default_rng(7)
    out = []
    for t, m in enumerate(pos):
        ids = np.array(sorted(m), dtype=np.int64)
        out.append(Term(f"T{t}", ids, np.array([max(1, len(m[d])) + int(rng.integers(0, 2)) for d in ids.tolist()], dtype=np.uint32)))
    return out


PHRASE_CASES = [  # (terms, slop, in_order)
    ((0, 1), 0, True), ((0, 1), 1, False), ((0, 1, 2), 0, False), ((0, 1, 2), 1, True), ((0, 1, 2), 3, False),
    ((2, 0, 1), 3, False), ((3, 4, 5, 6), 3, False), ((4, 3), None, True), (tuple(range(8)), 3, True),
    (tuple(range(8)), 8, False),
]


@pytest.fixture(scope="module")
def probe():
    return _probe()


@pytest.fixture(scope="module")
def lengths():
    return _lengths()


@pytest.fixture(scope="module")
def phrase_pos():
    return _phrase()


def _q(corpus, names):
    return [corpus[n] for n in names]


# ------------------------------------------------------------------------------------------------
# CPU: every class is reached, the checks reject wrong answers
# ------------------------------------------------------------------------------------------------
def test_probe_fixtures_reach_every_window_and_edge(probe):
    cl = {q: probe_classes(_q(probe, q[0]), q[1]) for q in PROBE_QUERIES}
    ab = cl[PROBE_QUERIES[0]]
    windows = [w for k in ab for w in k["windows"]]
    for w in (SMEM_ELEMS - 1, SMEM_ELEMS, SMEM_ELEMS + 1):
        assert w in windows, w
    assert max(windows) > 1_000_000
    assert [k for k in ab if SMEM_ELEMS + 1 in k["windows"] and not k["staged"][0]]
    assert [k for k in ab if SMEM_ELEMS in k["windows"] and k["staged"][0]]
    edges = set().union(*[k["edges"] for k in ab])
    assert {(0, "first"), (0, "last"), (0, "below"), (0, "above")} <= edges, edges
    surv = [k["survivors"] for k in ab]
    assert 0 in surv and CHUNK in surv and len(probe["A"].ids) % CHUNK
    assert any(surv[i] == 0 and surv[i - 1] == CHUNK and surv[i + 1] == CHUNK for i in range(1, len(surv) - 1))
    # the early exit with later NOT and OPTIONAL lists, survivors in the neighbouring CTAs
    for q in PROBE_QUERIES[1:3]:
        k = cl[q]
        ex = [i for i, x in enumerate(k) if x["early_exit"]]
        assert ex and all(k[i - 1]["survivors"] and k[i + 1]["survivors"] for i in ex), q
        assert {m for x in k for m in x["modes"]} == {0, 1, 2}
        e = set().union(*[x["edges"] for x in k])
        assert (1, "chunk_edge_member") in e and (2, "chunk_edge_member") in e, e
    # the empty NOT list, the OPTIONAL lists matching nothing and everything
    assert len(probe["E"].ids) == 0
    hits = and_expected(_q(probe, ("A", "B")), (0, 0))[0]
    assert not np.isin(hits, probe["O_none"].ids).any() and np.isin(hits, probe["O_all"].ids).all() and len(hits) > 5000
    for names, modes in PROBE_QUERIES:
        t = _q(probe, names)
        order = aggregate_order(t, modes)
        assert t[order[kernel_order(t, modes, order)[0]]].name == "A", names


def test_wide_fixtures_reach_every_child_count():
    w = _wide()
    for n in WIDE_NS:
        names, modes = wide_query(n)
        assert len(names) == n
        docs = and_expected(_q(w, names), modes)[0]
        assert len(docs) > 500, n
    assert len(w) - 2 == MAX_LISTS + 1  # 33 W lists: the refused AND


def test_length_fixtures_reach_every_scan_class(lengths):
    P = lengths["P"].ids
    for name in LENGTH_DRIVERS:
        t = _q(lengths, (name, "P"))
        order = aggregate_order(t, (0, 0))
        assert kernel_order(t, (0, 0), order)[0] == 0, name
    assert {len(lengths[n].ids) for n in LENGTH_DRIVERS} >= {1, 1023, 1024, 1025, 2048}
    D = lengths["D"].ids
    nch = n_chunks(len(D))
    assert nch > SCAN_ROUND and len(D) > SCAN_ROUND * CHUNK  # the scan carries across rounds
    counts = [int(np.isin(D[c * CHUNK:(c + 1) * CHUNK], P).sum()) for c in range(nch)]
    assert any(counts[i] == 0 and counts[i - 1] == CHUNK and counts[i + 1] for i in range(1, nch - 1))
    assert counts[SCAN_ROUND - 1] and 0 < sum(counts[SCAN_ROUND:])
    m = int(np.isin(D, P).sum())
    assert m > TOPN_WARPS * 1025 and all(len(evicting_ties(m, k)) == k - 1 for k in (32, 128, 129))


def test_masked_fixtures_drive_with_a_child_the_estimate_sorts_last():
    m = _masked()
    for q in MASK_QUERIES:
        t = _q(m, q)
        modes = (0,) * len(t)
        order = aggregate_order(t, modes)
        ko = kernel_order(t, modes, order)
        drv = order[ko[0]]
        assert t[drv].name.startswith("M") and order.index(drv) == len(t) - 1, q  # the driver sorts last by estimate
        assert ko != list(range(len(t))), q  # kernel slot != aggregate row
    assert MASK_CODEC["M2"][1] >> 64


def test_union_fixtures_reach_every_bitmap_edge_and_epoch():
    edge, u = _union_edges()
    docs = reduce(np.union1d, [u[f"E{c}"].ids for c in range(3)])
    words = {int(d) // 32 for d in edge}
    assert {0, 31, 32, 1023, 1024, 32767, 32768} <= words
    for w in (31, 32, 1023, 1024, 32767, 32768):
        assert 32 * w in docs and 32 * w + 31 in docs
    assert 0 not in docs and 1 in docs and 31 in docs
    assert int(docs[-1]) // 32 + 1 > 32 * 1024  # more than 1,024 32-word blocks: the block scan carries
    assert u["Etop"].ids[-1] == 0xFFFFFFFE and (0xFFFFFFFE // 32 + 1) * 4 == 512 << 20
    x = _union_exhaust()
    lasts = [int(x[f"X{c}"].ids[-1]) for c in range(5)]
    assert lasts[0] == lasts[1] and sorted(lasts[:4]) == [4999, 5000, 5000, 5001] and len(x["X5"].ids) == 0
    for n in (UNION_FLAT_MAX, UNION_FLAT_MAX + 1, MAX_LISTS, MAX_LISTS + 1):
        y = _union_many(n, n)
        cnt = sum(np.bincount(y[f"Y{c}"].ids, minlength=20_001) for c in range(n))
        assert cnt.max() <= 16 and (cnt >= 3).sum() > 500, n


def test_mask_and_numeric_fixtures_straddle_the_compaction_chunks():
    ids, fr, masks, filters = _mask_postings()
    keep = {k: np.flatnonzero(masks & f) for k, f in filters.items()}
    assert len(keep["none"]) == 0 and len(keep["all"]) == len(ids)
    per = np.bincount(keep["one_per_chunk"] // COMPACT_CHUNK)
    assert (per == 1).all() and len(per) == n_chunks(len(ids))
    assert {int(i) % COMPACT_CHUNK for i in keep["one_per_chunk"]} >= {0, 1023}
    assert keep["straddle"].tolist() == [3 * COMPACT_CHUNK - 1, 3 * COMPACT_CHUNK]
    nid, nv = _numeric_records()
    assert np.isinf(nv).any() and (np.signbit(nv) & (nv == 0)).any()
    nv = decoded_numeric(nid, nv)
    assert (np.diff(nid) >= 0).all()
    for b in range(1, 5):
        assert nid[b * COMPACT_CHUNK - 1] == nid[b * COMPACT_CHUNK], b
    # the first in-range record of a straddling document is on the left of a boundary for one range, on the right for another
    sides = set()
    P = ol.postings()
    for lo, hi, li, hi_i in NUMERIC_RANGES:
        for b in range(1, 5):
            i = b * COMPACT_CHUNK
            left, right = (P.orc_numeric_in_range(nv[i - 1], lo, hi, int(li), int(hi_i)), P.orc_numeric_in_range(nv[i], lo, hi, int(li), int(hi_i)))
            sides.add(("left" if left else "right") if (left or right) else "none")
    assert sides == {"left", "right", "none"}
    assert np.isinf(nv).any() and ((nv == 0) & ~np.signbit(nv)).any()


def test_phrase_fixtures_reach_every_position_class(phrase_pos):
    pos = phrase_pos
    deltas, zero_pos, zero_delta, empty, shared = set(), False, False, False, False
    for t, m in enumerate(pos):
        for d, p in m.items():
            empty |= not p
            zero_pos |= bool(p) and p[0] == 0
            zero_delta |= len(p) > 1 and 0 in np.diff(p)
            last = 0
            for x in p:
                deltas.add(varint_len(x - last))
                last = x
            shared |= t > 0 and bool(p) and any(x in pos[t - 1].get(d, []) for x in p)
    assert deltas == {1, 2, 3, 4, 5} and zero_pos and zero_delta and empty and shared
    assert max(max(p) for m in pos for p in m.values() if p) > 1 << 28
    # spans exactly at the slop and one above it, through the oracle's proximity check
    terms = _phrase_terms(pos)
    for names, slop, in_order in PHRASE_CASES:
        if slop is None:
            continue
        t = [terms[i] for i in names]
        docs, order, _ = and_expected(t, (0,) * len(t), in_order)
        offs = [[ol.varint_deltas(pos[names[c]][d]) for c in order] for d in docs.tolist()[:1500]]
        at = [ol.within_range(o, slop, in_order) for o in offs]
        below = [ol.within_range(o, slop - 1, in_order) if slop else False for o in offs]
        assert any(a and not b for a, b in zip(at, below)), (names, slop, in_order)  # span exactly slop
        above = [ol.within_range(o, slop + 1, in_order) for o in offs]
        assert any(b and not a for a, b in zip(at, above)), (names, slop, in_order)  # span exactly slop + 1


def test_the_checks_reject_a_dropped_hit_a_swapped_row_and_one_ulp(probe):
    t = _q(probe, ("A", "B", "O"))
    exp = and_expected(t, (0, 0, 2))
    docs, order, rows = exp
    check_set((docs, rows, order), exp, "itself")
    with pytest.raises(AssertionError):
        check_set((np.delete(docs, len(docs) // 2), rows[:, :-1], order), exp, "dropped hit")
    with pytest.raises(AssertionError):
        check_set((docs, rows[[1, 0, 2]], order), exp, "swapped rows")
    with pytest.raises(AssertionError):
        check_set((docs, rows, order[::-1]), exp, "child order")
    params = params_of(t)
    table = Table(np.random.default_rng(1))
    idx = np.arange(50)
    for scorer in ALL_SCORERS:
        s = expected_scores(scorer, docs, rows, order, params, table, idx, 2)
        check_scores(s, s, scorer, "itself")
        off = s.copy()
        off[7] = np.nextafter(off[7], np.inf) if scorer != ol.SCORER_BM25STD_TANH else off[7] + 4e-12 * max(1.0, abs(off[7]))
        with pytest.raises(AssertionError):
            check_scores(off, s, scorer, "one ulp")
    with pytest.raises(AssertionError):
        check_ranking(docs[:5][::-1], np.zeros(5), docs[:5], np.zeros(5), 5, "ties by docId")


def test_swapped_aggregate_rows_change_the_scores(probe):
    """the freq-row mutant of gather_kernel is visible in the scores as well as in the rows"""
    m = _masked()
    t = _q(m, MASK_QUERIES[1])
    docs, order, rows = and_expected(t, (0, 0, 0))
    params = params_of(t)
    table = Table(np.random.default_rng(2))
    idx = np.arange(min(300, len(docs)))
    for scorer in (ol.SCORER_BM25STD, ol.SCORER_TFIDF):
        good = expected_scores(scorer, docs, rows, order, params, table, idx, 2)
        bad = expected_scores(scorer, docs, rows[[1, 0, 2]], order, params, table, idx, 2)
        assert (good.view(np.uint64) != bad.view(np.uint64)).sum() > 100, scorer


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ps():
    from redisearch_b200 import postings

    return postings


@pytest.fixture(scope="module")
def table(ps):
    t = Table(np.random.default_rng(9))
    t.dt = ps.DocTable(N_DOCS, t.doc_len, t.doc_score, t.max_freq)
    return t


def launched(ps, fn, expected, what):
    """run fn and assert the chain's kernel launch count"""
    ps.stats(reset=True)
    out = fn()
    got = ps.stats().kernel_launches
    assert got == expected, f"{what}: {got} kernel launches, the per-query chain makes {expected}"
    return out


def upload(ps, terms):
    for t in terms.values():
        if getattr(t, "pl", None) is None:
            t.pl = ps.PostingList.from_arrays(t.ids.astype(np.uint64), t.freqs)
            assert len(t.pl) == len(t.ids)
    return terms


def _fetch_set(rs):
    ids, scores, fr = rs.fetch()
    return ids.astype(np.int64), scores, fr, rs.child_order().tolist()


def _check_and_scores(ps, rs, terms, modes, exp, table, scorers, what, extra=()):
    docs, order, rows = exp
    params = params_of(terms)
    idx = sample(len(docs), extra=extra)
    slop = max(1, len(terms) - 1)  # no term positions: GetSlop = children - 1, the virtual ones included
    for scorer in scorers:
        launched(ps, lambda: rs.score(scorer, params, agg_weight(scorer), N_DOCS, table.avg, getattr(table, "dt", None)),
                 L_SCORE if len(docs) else 0, (what, "score"))  # II_Score of an empty set launches nothing
        _, got, _, _ = _fetch_set(rs)
        check_scores(got[idx], expected_scores(scorer, docs, rows, order, params, table, idx, slop), scorer, (what, scorer))


@pytest.mark.gpu
def test_and_probe_windows_edges_and_early_exit(ps, probe, table):
    """intersect_kernel through II_IntersectEx: probe windows of 8,191 / 8,192 (staged) and 8,193 / over 1M entries (lower
    bound in global memory), driver entries on both ends of a window, below and above it, a CTA with no entry alive after the
    first probed list followed by NOT and OPTIONAL lists, NOT / OPTIONAL windows that begin or end on a chunk's edge entry, an
    empty NOT list, OPTIONAL lists matching nothing and everything; every scorer"""
    upload(ps, probe)
    for names, modes in PROBE_QUERIES:
        t = _q(probe, names)
        rs = launched(ps, lambda: ps.intersect_ex([x.pl for x in t], list(modes)), L_AND, names)
        exp = and_expected(t, modes)
        ids, _, fr, order = _fetch_set(rs)
        check_set((ids, fr, order), exp, names)
        _check_and_scores(ps, rs, t, modes, exp, table, ALL_SCORERS if names == ("A", "B", "N", "O") else (0, 2, 6), names)


@pytest.mark.gpu
def test_two_to_thirty_two_children_and_thirty_three_refused(ps, table):
    w = upload(ps, _wide())
    for n in WIDE_NS:
        names, modes = wide_query(n)
        t = _q(w, names)
        rs = launched(ps, lambda: ps.intersect_ex([x.pl for x in t], list(modes)), L_AND, n)
        exp = and_expected(t, modes)
        ids, _, fr, order = _fetch_set(rs)
        check_set((ids, fr, order), exp, n)
        _check_and_scores(ps, rs, t, modes, exp, table, (0, 1, 5, 6) if n == MAX_LISTS else (0, 2), n)
    over = [w[f"W{k}"].pl for k in range(MAX_LISTS + 1)]
    with pytest.raises(RuntimeError):
        launched(ps, lambda: ps.intersect_ex(over, [0] * len(over)), 0, "33 children")
    with pytest.raises(RuntimeError):
        ps.intersect(over)


@pytest.mark.gpu
def test_scan_and_gather_at_every_driver_length(ps, lengths, table):
    """drivers of 1, 1,023, 1,024, 1,025, 2,048 and 1,100,000 entries (the scan over 1,075 chunk counts carries into a second
    round), with chunks of zero survivors between full ones; II_Intersect and II_SearchTopN (chain: 5 launches)"""
    upload(ps, lengths)
    for name in LENGTH_DRIVERS:
        t = _q(lengths, (name, "P"))
        rs = launched(ps, lambda: ps.intersect([x.pl for x in t]), L_AND, name)
        exp = and_expected(t, (0, 0))
        ids, _, fr, order = _fetch_set(rs)
        check_set((ids, fr, order), exp, name)
        # the hits around the scan round boundary: the first survivor of chunk 1,024 of the driver
        D = t[0].ids
        extra = [int(np.searchsorted(exp[0], D[SCAN_ROUND * CHUNK]))] if len(D) > SCAN_ROUND * CHUNK else []
        _check_and_scores(ps, rs, t, (0, 0), exp, table, (0, 1), name, extra)
        params = params_of(t)
        sc = expected_scores(0, exp[0], exp[2], exp[1], params, table, np.arange(len(exp[0])), 1) if len(exp[0]) < 5000 else None
        gi, gs, total = launched(ps, lambda: ps.search_topn([x.pl for x in t], False, 0, params, AGG, N_DOCS, table.avg, table.dt, 100),
                                 L_SEARCH, (name, "search"))
        assert total == len(exp[0]), name
        if sc is not None:
            check_ranking(gi, gs, exp[0], sc, 100, name)


@pytest.mark.gpu
def test_driver_is_not_the_first_child_of_the_aggregate_order(ps, table):
    """field-mask-filtered children (FreqsFields; FreqsFieldsWide with a filter above bit 63) whose filtered length makes them
    the driver while their estimate sorts them last: freq rows at their aggregate row, the child order, BM25 / TFIDF bits that
    depend on it; II_SearchTopN and a batch at top_n 129 (the chain, not the fused route) rank like the oracle"""
    m = _masked()
    for name, t in m.items():
        if hasattr(t, "raw"):
            raw, fr, keep = t.raw
            codec, flt, dropped = MASK_CODEC[name]
            ix = ol.InvIndex(codec)
            for d, f, kp in zip(raw.tolist(), fr.tolist(), keep.tolist()):
                ix.add(d, f, (flt | 1) if kp else dropped)
            t.pl = launched(ps, lambda: ps.PostingList.from_blocks(ix.blocks(), codec, field_mask_filter=flt), L_FILTER, name)
            assert len(t.pl) == len(t.ids) and t.pl.num_estimated() == t.estimated
    upload(ps, m)
    for names in MASK_QUERIES:
        t = _q(m, names)
        modes = (0,) * len(t)
        rs = launched(ps, lambda: ps.intersect_ex([x.pl for x in t], list(modes)), L_AND, names)
        exp = and_expected(t, modes)
        ids, _, fr, order = _fetch_set(rs)
        check_set((ids, fr, order), exp, names)
        assert len(ids) > 200, names
        _check_and_scores(ps, rs, t, modes, exp, table, ALL_SCORERS, names)
        params = params_of(t)
        for scorer in (ol.SCORER_BM25, ol.SCORER_TFIDF):
            sc = expected_scores(scorer, exp[0], exp[2], exp[1], params, table, np.arange(len(exp[0])), max(1, len(t) - 1))
            gi, gs, total = launched(ps, lambda: ps.search_topn([x.pl for x in t], False, scorer, params, agg_weight(scorer), N_DOCS,
                                                                table.avg, table.dt, 50), L_SEARCH, (names, "search"))
            assert total == len(exp[0])
            check_ranking(gi, gs, exp[0], sc, 50, names)
            batch = ps.SearchBatch([([x.pl for x in t], params)], 129)
            got = launched(ps, lambda: batch.run(False, scorer, agg_weight(scorer), N_DOCS, table.avg, table.dt), L_SEARCH, (names, "batch 129"))
            assert got[0][2] == len(exp[0])
            check_ranking(got[0][0], got[0][1], exp[0], sc, 129, names)


def _union_expected(terms, quick=False):
    """docIds by union1d; per-child freq rows in the given (index) order; the reference's aggregate order of every hit from
    the oracle's UnionFlat (run_intersect)"""
    docs = reduce(np.union1d, [t.ids for t in terms])
    rows = freq_rows(terms, list(range(len(terms))), (0,) * len(terms), docs)
    return docs, rows


def _union_orders(terms, docs):
    idx = [ol.InvIndex(ol.CODEC_FREQS_ONLY, t.ids, t.freqs) for t in terms]
    hits = ol.run_intersect(idx, union=True)
    assert [h[0] for h in hits] == docs.tolist()
    return [[c for c, _ in ch] for _, ch in hits], hits


def _check_union(ps, terms, table, scorers, what, exact_order=True):
    n = len(terms)
    pls = [t.pl for t in terms]
    rs = launched(ps, lambda: ps.union(pls), union_launches(n) if any(len(t.ids) for t in terms) else 0, what)
    docs, rows = _union_expected(terms)
    ids, _, fr, order = _fetch_set(rs)
    if not len(docs):
        assert len(ids) == 0
        return
    check_set((ids, fr, order), (docs, list(range(n)), rows), what)
    quick = launched(ps, lambda: ps.union(pls, quick_exit=True), union_launches(n), (what, "quick"))
    assert quick.fetch(want_freqs=False)[0].astype(np.int64).tolist() == docs.tolist(), what
    params = params_of(terms)
    idx = sample(len(docs))
    if exact_order:
        orders, hits = _union_orders(terms, docs)
        for i in idx[:50].tolist():
            assert [f for _, f in hits[i][1]] == [int(rows[c, i]) for c in orders[i]], (what, i)
        order_of = lambda i: orders[i]
    else:
        order_of = lambda i: [c for c in range(n) if rows[c, i]]
    present = (rows != 0).sum(axis=0)
    slop = lambda i: max(1, int(present[i]) - 1)  # no term positions: GetSlop = present children - 1
    for scorer in scorers:
        launched(ps, lambda: rs.score(scorer, params, agg_weight(scorer), N_DOCS, table.avg, getattr(table, "dt", None)), L_SCORE,
                 (what, "score"))
        got = _fetch_set(rs)[1][idx]
        if scorer == ol.SCORER_DISMAX:  # a union's DISMAX is the best child's weight * freq (default.c:378-461): that child alone
            best = lambda i: [max(order_of(i), key=lambda c: params[c][0] * float(rows[c, i]))]
            exp = expected_scores(scorer, docs, lambda i: [rows[c, i] for c in best(i)], best, params, table, idx, slop)
        else:
            exp = expected_scores(scorer, docs, lambda i: [rows[c, i] for c in order_of(i)], order_of, params, table, idx, slop)
        if exact_order:
            check_scores(got, exp, scorer, (what, scorer))
        else:  # UnionHeap above 20 children: the sum's order follows the heap array (DESIGN §7)
            assert (np.abs(got - exp) <= 1e-13 * np.maximum(1.0, np.abs(exp))).all(), (what, scorer)
    return rs, docs


@pytest.mark.gpu
def test_union_bitmap_word_and_block_edges(ps, table):
    """docIds on the first and last bits of bitmap words 0, 31, 32, 1,023, 1,024, 32,767 and 32,768; every scorer"""
    edge, u = _union_edges()
    upload(ps, u)
    _check_union(ps, [u["E0"], u["E1"], u["E2"]], table, ALL_SCORERS, "edges")


@pytest.mark.gpu
def test_union_up_to_docid_0xfffffffe(ps):
    """the largest docId: the bitmap spans 2^27 words (512 MB, and as much again for the word offsets: fine on an 80 GB H100)
    and its block scan carries over 4,096 rounds; no doc table"""
    edge, u = _union_edges()
    upload(ps, u)
    _check_union(ps, [u["E0"], u["Etop"], u["E1"]], Table(), (0, 2, 6), "0xFFFFFFFE")


@pytest.mark.gpu
def test_union_children_running_out_together_and_empty_ones(ps, table):
    """children exhausted on the same docId and on neighbouring docIds (the UnionOrder epochs fix the scorer's summation
    order), a child empty from the start, and a union of empty lists only (no launch, no hit)"""
    x = upload(ps, _union_exhaust())
    _check_union(ps, [x[f"X{c}"] for c in range(6)], table, ALL_SCORERS, "exhaust")
    _check_union(ps, [x["X5"], x["X3"], x["X0"], x["X2"]], table, (0, 1, 6), "empty first")
    _check_union(ps, [x["X5"], x["X5"]], table, (), "all empty")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [UNION_FLAT_MAX, UNION_FLAT_MAX + 1, MAX_LISTS, MAX_LISTS + 1])
def test_union_of_20_21_32_and_33_children(ps, table, n):
    """20 children: the reference's UnionFlat, bit-exact; 21 and more: its UnionHeap (a documented deviation of the child order,
    DESIGN §7), 1e-13 relative; 33: the score tables move from the kernel arguments to device memory"""
    y = upload(ps, _union_many(n, n))
    _check_union(ps, [y[f"Y{c}"] for c in range(n)], table, (0, 1, 2, 6) if n <= UNION_FLAT_MAX else (0, 3, 6), n,
                 exact_order=n <= UNION_FLAT_MAX)


@pytest.mark.gpu
def test_topn_at_every_k_with_ties_across_warps(ps, lengths, table):
    """topn_kernel at k = 1, 128, 129, 1,000 and 1,024, the host partial sort at 1,025, fewer hits than k, and DOCSCORE with two
    doc scores: equal keys in every warp's list, ranked by docId"""
    upload(ps, lengths)
    t2 = Table(np.random.default_rng(4), two_scores=True)
    t2.dt = ps.DocTable(N_DOCS, t2.doc_len, t2.doc_score, t2.max_freq)
    big = _q(lengths, ("D", "P"))
    small = _q(lengths, ("L1025", "P"))  # fewer hits than k = 1,000 / 1,024 / 1,025: the device list is min(k, hits) long
    for terms, tab, scorer in ((big, t2, ol.SCORER_DOCSCORE), (small, table, ol.SCORER_BM25STD), (small, t2, ol.SCORER_DOCSCORE)):
        rs = ps.intersect([x.pl for x in terms])
        docs, order, rows = and_expected(terms, (0, 0))
        params = params_of(terms)
        rs.score(scorer, params, agg_weight(scorer), N_DOCS, tab.avg, tab.dt)
        if scorer == ol.SCORER_DOCSCORE:
            # DOCSCORE is the doc score: numpy for every hit, the oracle on a sample
            sc = tab.doc_score[docs].astype(np.float64)
            idx = sample(len(docs))
            check_scores(sc[idx], expected_scores(scorer, docs, rows, order, params, tab, idx, 1), scorer, "docscore")
            assert len(docs) > 8 * TOPN_WARPS * 1025 or len(docs) < 1000
        else:
            sc = expected_scores(scorer, docs, rows, order, params, tab, np.arange(len(docs)), 1)
        for k in (1, 128, 129, 1000, 1024, 1025, len(docs) + 5):
            gi, gs = launched(ps, lambda: rs.topn(k), L_TOPN if min(k, len(docs)) <= TOPN_DEVICE_MAX else 0, (scorer, k))
            assert len(gi) == min(k, len(docs))
            check_ranking(gi, gs, docs, sc, k, (scorer, k, len(docs)))


def topn_lists(m):
    """ii_topn_lists: 8 warps' lists per CTA, min(ceil(m / 256), 264) CTAs; warp g reads the 32-entry blocks g, g + lists, ..."""
    return TOPN_WARPS * min(-(-m // 256), 264)


def evicting_ties(m, k):
    """hit indices for doc score 1.0 among hits all at 0.5: k - 1 of warp 0's entries after its first k (its list is then full
    of equal keys), so that warp 0 has to evict k - 1 of them and keep exactly its smallest docId, the only 0.5 of the top k"""
    nw = topn_lists(m)
    warp0 = np.concatenate([np.arange(r * nw * 32, r * nw * 32 + 32) for r in range(-(-m // (nw * 32)))])
    warp0 = warp0[warp0 < m]
    assert len(warp0) >= 2 * k, (m, k)
    return warp0[k:2 * k - 1]


@pytest.mark.gpu
def test_topn_evicts_the_largest_docid_of_equal_keys(ps, lengths):
    """topn_kernel's list replacement: with every kept key equal, the entry evicted is the one with the largest docId"""
    upload(ps, lengths)
    terms = _q(lengths, ("D", "P"))
    rs = ps.intersect([x.pl for x in terms])
    docs = and_expected(terms, (0, 0))[0]
    for k in (32, 128, 129):
        score = np.full(N_DOCS + 1, 0.5, dtype=np.float32)
        score[docs[evicting_ties(len(docs), k)]] = 1.0
        dt = ps.DocTable(N_DOCS, None, score, None)
        rs.score(ol.SCORER_DOCSCORE, params_of(terms), AGG, N_DOCS, 250.0, dt)
        gi, gs = launched(ps, lambda: rs.topn(k), L_TOPN, k)
        check_ranking(gi, gs, docs, score[docs].astype(np.float64), k, k)
        assert gi[-1] == docs[0], k


@pytest.mark.gpu
def test_mask_compaction_keeps_none_all_or_one_per_chunk(ps):
    """mask_flags / mask_compact (FreqsFields and FreqsFieldsWide): filters keeping no posting, all of them, exactly one per
    1,024-entry chunk (at its first, last and inner offsets) and the two postings either side of a chunk boundary"""
    ids, fr, masks, filters = _mask_postings()
    for codec in (ol.CODEC_FREQS_FIELDS, ol.CODEC_FREQS_FIELDS_WIDE):
        ix = ol.InvIndex(codec)
        for d, f, mk in zip(ids.tolist(), fr.tolist(), masks.tolist()):
            ix.add(d, f, mk)
        blocks = ix.blocks()
        for what, flt in filters.items():
            pl = launched(ps, lambda: ps.PostingList.from_blocks(blocks, codec, field_mask_filter=flt), L_FILTER, (codec, what))
            keep = (masks & flt) != 0
            assert len(pl) == int(keep.sum()) and pl.num_estimated() == len(ids), (codec, what)
            if keep.any():
                got, _, gf = ps.union([pl]).fetch()
                assert got.astype(np.int64).tolist() == ids[keep].tolist() and gf[0].tolist() == fr[keep].tolist(), (codec, what)


@pytest.mark.gpu
def test_numeric_compaction_at_chunk_boundaries_and_infinities(ps):
    """numeric_flags / numeric_compact: multi-value documents whose records straddle each 1,024 boundary, with the first
    in-range record on either side; ranges at +-inf and -0.0 with inclusive and exclusive ends"""
    nid, raw = _numeric_records()
    nl = ps.NumericList(ol.numeric_blocks(nid.tolist(), raw.tolist()))
    nv = decoded_numeric(nid, raw)
    got_ids, got_vals = nl.fetch()
    assert got_ids.astype(np.int64).tolist() == nid.tolist() and got_vals.tobytes() == nv.tobytes()
    for lo, hi, li, hi_i in NUMERIC_RANGES:
        exp = expected_numeric(nid, nv, lo, hi, li, hi_i)
        pl = launched(ps, lambda: nl.filter(lo, hi, li, hi_i), L_FILTER, (lo, hi, li, hi_i))
        assert len(pl) == len(exp), (lo, hi, li, hi_i)
        if len(exp):
            got, _, gf = ps.union([pl]).fetch()
            assert got.astype(np.int64).tolist() == exp.tolist() and (gf[0] == 1).all(), (lo, hi, li, hi_i)


def _phrase_lists(ps, pos):
    terms = _phrase_terms(pos)
    idx = []
    for t, term in enumerate(terms):
        ix = ol.InvIndex(ol.CODEC_FULL)
        for d, f in zip(term.ids.tolist(), term.freqs.tolist()):
            ix.add(d, f, 1, ol.varint_deltas(pos[t][d]))
        idx.append(ix)
    pls = ps.postings_with_offsets([ix.blocks() for ix in idx], ol.CODEC_FULL)
    for term, pl in zip(terms, pls):
        term.pl = pl
    return terms


@pytest.mark.gpu
def test_phrase_filter_and_getslop_over_crafted_positions(ps, phrase_pos, table):
    """phrase_filter_kernel + flag_compact through II_IntersectPhrase (in order and not, 2 to 8 children, 9 refused) and
    min_offset_delta_kernel through the legacy scorers: varints of 1 to 5 bytes, position 0, zero deltas, overlapping positions,
    spans of exactly the slop and one more, records without positions inside a hit"""
    pos = phrase_pos
    terms = _phrase_lists(ps, pos)
    for names, slop, in_order in PHRASE_CASES:
        t = [terms[i] for i in names]
        modes = (0,) * len(t)
        rs = launched(ps, lambda: ps.intersect_phrase([x.pl for x in t], slop, in_order), L_PHRASE, (names, slop, in_order))
        docs, order, _ = and_expected(t, modes, in_order)
        docs = np.array([d for d in docs.tolist() if ol.within_range([ol.varint_deltas(pos[names[c]][d]) for c in order], slop, in_order)],
                        dtype=np.int64)
        rows = freq_rows(t, order, modes, docs)
        ids, _, fr, got_order = _fetch_set(rs)
        check_set((ids, fr, got_order), (docs, order, rows), (names, slop, in_order))
        assert len(docs) > 20, (names, slop, in_order)
        params = params_of(t)
        idx = sample(len(docs), limit=3000)
        slops = np.array([ol.min_offset_delta([pos[names[c]][int(docs[i])] for c in order]) for i in idx.tolist()])
        for scorer in LEGACY:
            launched(ps, lambda: rs.score(scorer, params, agg_weight(scorer), N_DOCS, table.avg, table.dt), L_SCORE + L_SLOP * (scorer == LEGACY[0]),
                     (names, scorer))
            got = _fetch_set(rs)[1][idx]
            exp = expected_scores(scorer, docs, rows, order, params, table, idx, lambda i: int(slops[np.searchsorted(idx, i)]))
            check_scores(got, exp, scorer, (names, slop, in_order, scorer))
    nine = [terms[i % PHRASE_MAX_LISTS].pl for i in range(PHRASE_MAX_LISTS + 1)]
    with pytest.raises(RuntimeError):
        launched(ps, lambda: ps.intersect_phrase(nine, 3, True), 0, "9 children")


@pytest.mark.gpu
def test_phrase_over_a_nested_union_with_duplicate_positions(ps, phrase_pos):
    """merge_write_kernel: a nested OR (T1 | T2) whose merged position stream repeats positions both terms hold, inside a
    phrase with T0 and T3; the nested child's freq is the sum of its children's"""
    pos = phrase_pos
    terms = _phrase_lists(ps, pos)
    T0, T1, T2, T3 = terms[0], terms[1], terms[2], terms[3]
    inner = ps.union([T1.pl, T2.pl])
    nested = inner.into_child(params_of([T1, T2]), 1.0, with_positions=True)
    ids12 = np.union1d(T1.ids, T2.ids)
    merged = {d: sorted(pos[1].get(d, []) + pos[2].get(d, [])) for d in ids12.tolist()}
    dup = sum(len(v) != len(set(v)) for v in merged.values())
    assert dup > 100
    f12 = freq_rows([T1, T2], [0, 1], (0, 0), ids12).sum(axis=0).astype(np.uint32)
    NT = Term("T1|T2", ids12, f12, estimated=T1.estimated + T2.estimated)
    NT.pl = nested
    t = [T0, NT, T3]

    def node(c, d):
        """the hit's result tree node of child c: a term leaf, or the OR of the terms present (the oracle merges its positions)"""
        if c != 1:
            return {"kind": ol.KIND_TERM, "positions": pos[3 if c == 2 else 0][d]}
        return {"kind": ol.KIND_OR, "children": [{"kind": ol.KIND_TERM, "positions": pos[k][d]} for k in (1, 2) if d in pos[k]]}

    for slop, in_order in ((0, True), (2, False), (1, True)):
        rs = launched(ps, lambda: ps.intersect_phrase([x.pl for x in t], slop, in_order), L_PHRASE, (slop, in_order))
        docs, order, _ = and_expected(t, (0, 0, 0), in_order)
        docs = np.array([d for d in docs.tolist()
                         if ol.ResultTree({"kind": ol.KIND_AND, "children": [node(c, d) for c in order]}).within_range(slop, in_order)],
                        dtype=np.int64)
        ids, _, fr, got_order = _fetch_set(rs)
        check_set((ids, fr, got_order), (docs, order, freq_rows(t, order, (0, 0, 0), docs)), (slop, in_order))
        assert len(docs) > 20
