"""Compound hybrid pre-filters — ANDs over pending ORs and numeric ranges — on the device, feeding the device KNN batch
(DESIGN.md §4.8): prints one JSON line.

Workload: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest), k = 10, batches of 16 and 256 queries, and
three filter shapes over bench_hybrid_filters' synthetic 50M-doc Zipf posting lists and its 128-leaf price field:
  term_tag        `@brand:x @category:{a|b|...}`: a term of rank 20..99 AND an OR of 4-50 terms of ranks 100..1099
  term_price      `@brand:x @price:[lo hi]`: a term of rank 20..99 AND a range of 0.1 % or 1 % of the prices
  tag_price_not   `@category:{...} @price:[lo hi] -@tag:{...}`: an OR of 4-50 terms AND a range AND NOT an OR of 4 terms
Per (shape, queries per batch) the line reports:
  host_path_ms    today's best: II_UnionBatchDevice / II_NumericFilterBatchDevice, then per set II_ResultSet_Len and
                  II_PostingList_FromDevice, then II_IntersectBatchDevice (II_IntersectEx per query for the NOT shape, which
                  II_IntersectBatchDevice cannot express), then one VecSimB200_TopKFilteredBatchDevice; wall clock per batch up to
                  the stream's completion, median of --steps
  device_path_ms  the same filter batches, II_IntersectFilterBatchDevice, the same KNN and II_ResultSet_FreeAfter on one stream,
                  with no host wait; wall clock per batch up to the stream's completion, median of --steps
  launches        posting-list kernels (II_GetStats, plus II_IntersectBatchDevice's 3 per AND on its own streams) and vector
                  kernels (VecSimB200_GetStats) of one batch on each path
  and_ms          device time of the three ifb_* kernels of one device-path batch (torch.profiler, a run of its own) and the bytes
                  they move at least (every driver docId read once; every survivor written to scratch, read back and written out)
                  against the 3.35 TB/s data-sheet HBM3 peak of the H100 SXM
and parity of 8 device-path answers (4 term_price, 4 tag_price_not) against the reference's distance kernel (oracle/_ref when
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

PEAK_GBS = 3350.0  # H100 SXM data sheet
TERM_RANKS = range(20, 100)
K = 10
AND_KERNELS = ("ifb_probe", "ifb_scan", "ifb_expand")


def log(msg):
    print(f"[bench_hybrid_compound {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


class _NoSet:
    """the host path's stand-in for an AND that built no set: nothing to free"""

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

    rng = np.random.default_rng(5)
    result, parity = {}, {}
    for nq in (16, 256):
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0  # stored form: normalised
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qdev.cpu().numpy())

        def tag_or(lo, hi):
            return [lists[r] for r in rng.choice(list(TAG_RANKS), int(rng.integers(lo, hi + 1)), replace=False).tolist()]

        def price_range(i):
            span = len(sorted_prices) // (1000 if i % 2 == 0 else 100)
            a = int(rng.integers(0, len(sorted_prices) - span))
            lo, hi = float(sorted_prices[a]), float(sorted_prices[a + span])
            return ([leaves[j] for j, (mn, mx) in enumerate(leaf_bounds) if mx >= lo and mn <= hi], lo, hi, 1, 1)  # the tree walk's leaves

        term = lambda: lists[int(rng.choice(list(TERM_RANKS)))]  # noqa: E731
        shapes = {  # per query: (terms, ORs, ranges, [(kind, index, mode)]) with kind t / o / p
            "term_tag": [([term()], [tag_or(4, 50)], [], [("t", 0, 0), ("o", 0, 0)]) for _ in range(nq)],
            "term_price": [([term()], [], [price_range(i)], [("t", 0, 0), ("p", 0, 0)]) for i in range(nq)],
            "tag_price_not": [([], [tag_or(4, 50), tag_or(4, 4)], [price_range(i)], [("o", 0, 0), ("p", 0, 0), ("o", 1, 1)]) for i in range(nq)],
        }
        out_l = torch.empty((nq, K), dtype=torch.int64, device=dev)
        out_s = torch.empty((nq, K), dtype=torch.float32, device=dev)
        out_c = torch.empty(nq, dtype=torch.int32, device=dev)
        host_keep, pool_launches = [], [0]
        for shape, qs in shapes.items():
            has_not = any(m for q in qs for *_, m in q[3])

            def filter_sets(s):
                """the ORs and ranges of every query as pending sets: per query (or sets, range sets), and every set"""
                ors = [o for q in qs for o in q[1]]
                rngs = [p for q in qs for p in q[2]]
                o_sets = ps.union_batch_device(ors, quick_exit=True, stream=s) if ors else []
                p_sets = ps.numeric_filter_batch_device(rngs, stream=s) if rngs else []
                per_q, io, ip = [], 0, 0
                for q in qs:
                    per_q.append(([r[0] for r in o_sets[io:io + len(q[1])]], [r[0] for r in p_sets[ip:ip + len(q[2])]]))
                    io += len(q[1])
                    ip += len(q[2])
                return per_q, [r[0] for r in o_sets + p_sets if r[0] is not None]

            def knn(sets, extra):
                rc = index.topk_filtered_batch_device(qdev, K, [r[1] for r in sets], [r[3] for r in sets], counts=[r[2] for r in sets],
                                                      out_labels=out_l, out_scores=out_s, out_counts=out_c, stream=stream)[3]
                for rs in [r[0] for r in sets] + extra:
                    if rs is not None:
                        rs.free_after(stream)
                return rc

            def device_ands():
                per_q, inputs = filter_sets(stream)
                batch = [[(q[0][i] if k == "t" else per_q[n][0][i] if k == "o" else per_q[n][1][i], m) for k, i, m in q[3]]
                         for n, q in enumerate(qs)]
                return ps.intersect_filter_batch_device(batch, stream=stream), inputs

            def device_path():
                sets, inputs = device_ands()
                return knn(sets, inputs)

            def host_ands():
                per_q, inputs = filter_sets(stream)
                views, out = [], []
                for n, q in enumerate(qs):
                    kids = []
                    for k, i, m in q[3]:
                        if k == "t":
                            kids.append(q[0][i])
                            continue
                        rs = per_q[n][0][i] if k == "o" else per_q[n][1][i]
                        c = len(rs)  # the host wait of this path
                        assert c <= len(ones)
                        kids.append(ps.PostingList(P.II_PostingList_FromDevice(P.II_ResultSet_DeviceDocIds(rs.h), ones.data_ptr(), c)))
                    views.append(kids)
                if has_not:  # II_IntersectBatchDevice takes no NOT children
                    for q, kids in zip(qs, views):
                        rs = ps.intersect_ex(kids, [m for *_, m in q[3]])
                        m = len(rs)
                        out.append((rs, P.II_ResultSet_DeviceDocIds(rs.h) if m else None, P.II_ResultSet_DeviceLen(rs.h), m, None))
                else:
                    out = [r + (None,) for r in ps.intersect_batch_device(views, stream=stream)]
                    # II_IntersectBatchDevice counts its 3 launches per AND on its own contexts, not the caller's
                    pool_launches[0] = 3 * sum(r[0] is not None for r in out)
                return out, inputs, views

            def host_path():
                sets, inputs, views = host_ands()
                host_keep[:] = [views]  # the list views live until the next batch: II_IntersectBatchDevice reads them on its streams
                return knn([r[:4] for r in sets], inputs)

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
                pool_launches[0] = 0
                assert call() == 0
                stream.synchronize()
                launches[name] = {"filters": int(ps.stats(reset=True).kernel_launches) + pool_launches[0],
                                  "knn": int(index.stats(reset=True).kernel_launches)}
            r["launches"] = launches
            # the AND kernels' device time, and the bytes they move at least
            from torch.profiler import ProfilerActivity, profile

            per_q, inputs = filter_sets(stream)
            stream.synchronize()
            batch = [[(q[0][i] if k == "t" else per_q[n][0][i] if k == "o" else per_q[n][1][i], m) for k, i, m in q[3]] for n, q in enumerate(qs)]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                sets = ps.intersect_filter_batch_device(batch, stream=stream)
                stream.synchronize()
            and_us = sum(ev.device_time_total for ev in prof.key_averages()
                         if any(k in ev.key for k in AND_KERNELS) and getattr(ev, "device_time_total", 0) > 0)
            hits = sum(len(x[0]) for x in sets if x[0] is not None)
            driver = 0
            for q in batch:  # the driver: the required child with the smallest host bound; its count on the device
                req = [c for c, m in q if m == 0]
                bounds = [len(c) if isinstance(c, ps.PostingList) else P.II_ResultSet_Capacity(c.h) for c in req]
                driver += len(req[int(np.argmin(bounds))])
            moved = 4 * driver + 12 * hits
            for x in sets:
                if x[0] is not None:
                    x[0].close()
            for rs in inputs:
                rs.close()
            r["and_ms"] = and_us / 1000.0
            r["and_driver_entries"] = int(driver)
            r["and_hits"] = int(hits)
            r["and_bytes"] = int(moved)
            r["and_GBs"] = moved / (and_us * 1e-6) / 1e9 if and_us else None
            r["and_frac_of_peak"] = r["and_GBs"] / PEAK_GBS if r["and_GBs"] else None
            result[f"{shape}_nq{nq}_k{K}"] = r
            log(f"{shape} nq={nq}: {r}")
            if not args.no_parity and nq == 16 and shape in ("term_price", "tag_price_not"):
                assert device_path() == 0
                stream.synchronize()
                dl, dsc, dc = out_l.cpu().numpy(), out_s.cpu().numpy(), out_c.cpu().numpy()
                host_sets, host_inputs, _views = host_ands()
                stream.synchronize()
                # an AND with an empty child is no set (cap 0, skipped by the check): a stand-in keeps the rows aligned with the queries
                host_sets = [r if r[0] is not None else (_NoSet(),) + tuple(r[1:]) for r in host_sets]
                parity[shape] = check_parity(env, index, total, host_sets, qh, dl, dsc, dc)
                for rs in host_inputs:
                    rs.close()
    print(json.dumps({
        "metric": "hybrid filtered-KNN batches with compound (AND over OR / numeric-range) pre-filters on the device",
        "unit": "ms per batch", "card": card(), "corpus": {"rows": total, "dim": DIM, "dtype": "f32", "metric": "cosine", "data": "synthetic"},
        "filters": {"term_tag": f"a term of ranks {TERM_RANKS.start}..{TERM_RANKS.stop - 1} AND an OR of 4-50 terms of ranks "
                                f"{TAG_RANKS.start}..{TAG_RANKS.stop - 1}, synthetic Zipf over {POSTINGS_DOCS} docs",
                    "term_price": "the same terms AND 0.1 % / 1 % price ranges (bench_hybrid_filters' price field)",
                    "tag_price_not": "an OR of 4-50 terms AND a price range AND NOT an OR of 4 terms"},
        "k": K, "steps": args.steps, "warmup": args.warmup, "peak_GBs": PEAK_GBS, "results": result, "parity": parity or None}))
    env.close()


if __name__ == "__main__":
    main()
