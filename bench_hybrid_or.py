"""ORs over pending filter sets — ANDs and numeric ranges — on the device, feeding the device KNN batch (DESIGN.md §4.9): prints
one JSON line.

Workload: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest), k = 10, batches of 16 and 256 queries, and
three filter shapes over bench_hybrid_filters' synthetic 50M-doc Zipf posting lists and its 128-leaf price field:
  and_or_and        `(@brand:x @color:y) | (@brand:z @color:w)`: two ANDs of a term of rank 20..99 and a tag of rank 100..1099
  price_bands       `@price:[a b] | @price:[c d]`: two ranges of 0.1 % of the prices each
  tagprice_or_term  `(@category:{x} @price:[a b]) | @brand:y`: a tag AND a 0.1 % range, OR a term of rank 20..99
The child sets come from the same batch calls on both paths: II_NumericFilterBatchDevice for the ranges, then
II_IntersectFilterBatchDevice for the ANDs.  Per (shape, queries per batch) the line reports:
  host_path_ms    the child batches, then per set II_ResultSet_Len and II_PostingList_FromDevice, then II_UnionBatchDevice(quick),
                  then one VecSimB200_TopKFilteredBatchDevice; wall clock per batch up to the stream's completion, median of --steps
  device_path_ms  the child batches, II_UnionFilterBatchDevice, the same KNN and II_ResultSet_FreeAfter on one stream, with no host
                  wait; wall clock per batch up to the stream's completion, median of --steps
  launches        posting-list kernels (II_GetStats) and vector kernels (VecSimB200_GetStats) of one batch on each path
  or_ms           device time of the four ub_* kernels of one II_UnionFilterBatchDevice call (torch.profiler, a run of its own)
and parity of 8 device-path answers (4 price_bands, 4 tagprice_or_term) against the reference's distance kernel (oracle/_ref when
built, else the C restatement) over the filtered rows read back with VecSimB200_ReadRows, in (distance, docId) order.  The card
name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, N_ROWS, SEED_QUERIES, Env, build_shard  # noqa: E402
from bench_hybrid_filters import POSTINGS_DOCS, TAG_RANKS, check_parity, price_leaves  # noqa: E402
from bench_int8_l2 import card  # noqa: E402

TERM_RANKS = range(20, 100)
K = 10
OR_KERNELS = ("ub_mark", "ub_popc", "ub_scan", "ub_expand")


def log(msg):
    print(f"[bench_hybrid_or {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


class _NoSet:
    """the host path's stand-in for an OR that built no set: nothing to free"""

    def close(self):
        pass


def main():
    import numpy as np

    from redisearch_b200 import postings as ps
    from redisearch_b200._lib import load_library

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()
    torch, vs = env.torch, env.vs
    total, dev, sp, stream = args.rows, env.dev, env.sp, env.stream
    t0 = time.perf_counter()
    index, _ = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, total, 0)
    log(f"corpus built in {time.perf_counter() - t0:.1f} s")

    S = load_library("libsynth_b200.so")
    S.Synth_DocFreq.restype = C.c_uint64
    S.Synth_DocFreq.argtypes = [C.c_uint64, C.c_uint64]
    S.Synth_Postings.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    P = ps.lib()
    chunks = (POSTINGS_DOCS + 1023) // 1024
    scratch = torch.empty(2 * chunks + 16, dtype=torch.int32, device=dev)
    d_total = torch.zeros(4, dtype=torch.int32, device=dev)
    h_count = np.zeros(4, dtype=np.uint32)
    lists = {}
    for r in list(TERM_RANKS) + list(TAG_RANKS):
        cap = int(S.Synth_DocFreq(POSTINGS_DOCS, r) * 1.2) + 4096
        ids = torch.empty(cap, dtype=torch.int32, device=dev)
        fr = torch.empty(cap, dtype=torch.int32, device=dev)
        assert S.Synth_Postings(POSTINGS_DOCS, r, ids.data_ptr(), fr.data_ptr(), scratch.data_ptr(), d_total.data_ptr(), h_count.ctypes.data, sp) == 0
        lists[r] = ps.PostingList(P.II_PostingList_FromDevice(ids.data_ptr(), fr.data_ptr(), int(h_count[0])))
        del ids, fr
    # freqs of the host path's list views: as many as the largest set can hold (every docId of the synthetic lists)
    ones = torch.ones(POSTINGS_DOCS + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    leaves, leaf_bounds, sorted_prices = price_leaves(np, ps, total)
    log(f"{len(lists)} posting lists and {len(leaves)} price leaves built")

    rng = np.random.default_rng(9)
    result, parity = {}, {}
    for nq in (16, 256):
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0  # stored form: normalised
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qdev.cpu().numpy())

        def price_range():
            span = len(sorted_prices) // 1000
            a = int(rng.integers(0, len(sorted_prices) - span))
            lo, hi = float(sorted_prices[a]), float(sorted_prices[a + span])
            return ([leaves[j] for j, (mn, mx) in enumerate(leaf_bounds) if mx >= lo and mn <= hi], lo, hi, 1, 1)  # the tree walk's leaves

        term = lambda: lists[int(rng.choice(list(TERM_RANKS)))]  # noqa: E731
        tag = lambda: lists[int(rng.choice(list(TAG_RANKS)))]  # noqa: E731
        # per query: (ranges, ANDs, OR children); an AND child is ("t", list) or ("p", range index), an OR child ("t", list),
        # ("a", AND index) or ("p", range index)
        shapes = {
            "and_or_and": [([], [[("t", term()), ("t", tag())], [("t", term()), ("t", tag())]], [("a", 0), ("a", 1)]) for _ in range(nq)],
            "price_bands": [([price_range(), price_range()], [], [("p", 0), ("p", 1)]) for _ in range(nq)],
            "tagprice_or_term": [([price_range()], [[("t", tag()), ("p", 0)]], [("a", 0), ("t", term())]) for _ in range(nq)],
        }
        out_l = torch.empty((nq, K), dtype=torch.int64, device=dev)
        out_s = torch.empty((nq, K), dtype=torch.float32, device=dev)
        out_c = torch.empty(nq, dtype=torch.int32, device=dev)
        host_keep = []
        for shape, qs in shapes.items():

            def child_sets(s):
                """the ranges, then the ANDs, of every query as pending sets: per query (AND sets, range sets), and every set"""
                rngs = [p for q in qs for p in q[0]]
                p_sets = [r[0] for r in ps.numeric_filter_batch_device(rngs, stream=s)] if rngs else []
                per_p, ip = [], 0
                for q in qs:
                    per_p.append(p_sets[ip:ip + len(q[0])])
                    ip += len(q[0])
                ands = [[(x if k == "t" else per_p[n][x], 0) for k, x in a] for n, q in enumerate(qs) for a in q[1]]
                a_sets = [r[0] for r in ps.intersect_filter_batch_device(ands, stream=s)] if ands else []
                per_q, ia = [], 0
                for n, q in enumerate(qs):
                    per_q.append((a_sets[ia:ia + len(q[1])], per_p[n]))
                    ia += len(q[1])
                return per_q, [rs for rs in a_sets + p_sets if rs is not None]

            def or_batch(per_q):
                return [[x if k == "t" else per_q[n][0][x] if k == "a" else per_q[n][1][x] for k, x in q[2]] for n, q in enumerate(qs)]

            def knn(sets, extra):
                rc = index.topk_filtered_batch_device(qdev, K, [r[1] for r in sets], [r[3] for r in sets], counts=[r[2] for r in sets],
                                                      out_labels=out_l, out_scores=out_s, out_counts=out_c, stream=stream)[3]
                for rs in [r[0] for r in sets] + extra:
                    if rs is not None:
                        rs.free_after(stream)
                return rc

            def device_path():
                per_q, inputs = child_sets(stream)
                return knn(ps.union_filter_batch_device(or_batch(per_q), stream=stream), inputs)

            def host_ors():
                per_q, inputs = child_sets(stream)
                views = []
                for kids in or_batch(per_q):
                    v = []
                    for c in kids:
                        if isinstance(c, ps.PostingList):
                            v.append(c)
                        elif c is not None:
                            m = len(c)  # the host wait of this path
                            assert m <= len(ones)
                            if m:
                                v.append(ps.PostingList(P.II_PostingList_FromDevice(P.II_ResultSet_DeviceDocIds(c.h), ones.data_ptr(), m)))
                    views.append(v)
                return ps.union_batch_device(views, quick_exit=True, stream=stream), inputs, views

            def host_path():
                sets, inputs, views = host_ors()
                host_keep[:] = [views]  # the list views live until the next batch
                return knn(sets, inputs)

            def timed(call):
                ms = []
                for _ in range(args.steps):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    assert call() == 0
                    stream.synchronize()
                    ms.append((time.perf_counter() - t) * 1000.0)
                return float(np.median(ms))

            for _ in range(max(1, args.warmup)):
                assert device_path() == 0 and host_path() == 0
            torch.cuda.synchronize()
            r = {"device_path_ms": timed(device_path), "host_path_ms": timed(host_path)}
            r["speedup"] = r["host_path_ms"] / r["device_path_ms"]
            launches = {}
            for name, call in (("device_path", device_path), ("host_path", host_path)):
                torch.cuda.synchronize()
                ps.stats(reset=True)
                index.stats(reset=True)
                assert call() == 0
                stream.synchronize()
                launches[name] = {"filters": int(ps.stats(reset=True).kernel_launches), "knn": int(index.stats(reset=True).kernel_launches)}
            r["launches"] = launches
            # the OR kernels' device time, in a run of its own (the child batches run first and are not in the window)
            from torch.profiler import ProfilerActivity, profile

            per_q, inputs = child_sets(stream)
            batch = or_batch(per_q)
            stream.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                sets = ps.union_filter_batch_device(batch, stream=stream)
                stream.synchronize()
            or_us = sum(ev.device_time_total for ev in prof.key_averages()
                        if any(k in ev.key for k in OR_KERNELS) and getattr(ev, "device_time_total", 0) > 0)
            r["or_ms"] = or_us / 1000.0
            r["or_hits"] = int(sum(len(x[0]) for x in sets if x[0] is not None))
            for x in sets:
                if x[0] is not None:
                    x[0].close()
            for rs in inputs:
                rs.close()
            result[f"{shape}_nq{nq}_k{K}"] = r
            log(f"{shape} nq={nq}: {r}")
            if not args.no_parity and nq == 16 and shape in ("price_bands", "tagprice_or_term"):
                assert device_path() == 0
                stream.synchronize()
                dl, dsc, dc = out_l.cpu().numpy(), out_s.cpu().numpy(), out_c.cpu().numpy()
                host_sets, host_inputs, _views = host_ors()
                stream.synchronize()
                # an OR with no child set builds no set (cap 0, skipped by the check): a stand-in keeps the rows aligned with the queries
                host_sets = [(x[0], x[1], x[2], len(x[0]), None) if x[0] is not None else (_NoSet(), None, None, 0, None) for x in host_sets]
                parity[shape] = check_parity(env, index, total, host_sets, qh, dl, dsc, dc)
                for rs in host_inputs:
                    rs.close()
    print(json.dumps({
        "metric": "hybrid filtered-KNN batches with ORs over pending AND / numeric-range pre-filters on the device",
        "unit": "ms per batch", "card": card(), "corpus": {"rows": total, "dim": DIM, "dtype": "f32", "metric": "cosine", "data": "synthetic"},
        "filters": {"and_or_and": f"(a term of ranks {TERM_RANKS.start}..{TERM_RANKS.stop - 1} AND a tag of ranks {TAG_RANKS.start}.."
                                  f"{TAG_RANKS.stop - 1}) OR (the same), synthetic Zipf over {POSTINGS_DOCS} docs",
                    "price_bands": "a 0.1 % price range OR another (bench_hybrid_filters' price field)",
                    "tagprice_or_term": "(a tag AND a 0.1 % price range) OR a term"},
        "k": K, "steps": args.steps, "warmup": args.warmup, "results": result, "parity": parity or None}))
    env.close()


if __name__ == "__main__":
    main()
