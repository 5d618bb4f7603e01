"""Batches of OR and numeric-range pre-filters on the device, feeding the device KNN batch (DESIGN.md §4.7): prints one JSON line.

Workload: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest) and two filter shapes per batch of 16 and
256 queries:
  tag     ORs of 4-200 terms (`@tag:{a|b|...}`) over the synthetic 50M-doc Zipf posting lists of bench_postings (libsynth_b200),
          term ranks 100..1099
  price   ranges of 0.1 % and 1 % of the values (`@price:[lo hi]`, half each) of a synthetic price field of 2M documents (every
          5th docId, 1 % of them with a second price), split by value into 128 leaves as a range tree splits it; the leaves a
          range overlaps are the ones the host's tree walk picks
Per (shape, queries per batch), k = 10, the line reports:
  host_path_ms    per query II_Union(quick) (price: II_NumericList_Filter of each leaf first), II_ResultSet_Len, then one
                  VecSimB200_TopKFilteredBatchDevice; wall clock per batch up to the stream's completion, median of --steps
  device_path_ms  II_UnionBatchDevice / II_NumericFilterBatchDevice + VecSimB200_TopKFilteredBatchDevice + II_ResultSet_FreeAfter
                  on one stream, wall clock per batch up to the stream's completion, median of --steps
  launches        posting-list kernels (II_GetStats) and vector kernels (VecSimB200_GetStats) of one batch on each path
  filter_ms       device time of the filter kernels of one device-path batch (torch.profiler) and the bytes they move at least
                  (postings read, values read for price, bitmap cleared / marked / counted / expanded, docIds written) against the
                  3.35 TB/s data-sheet HBM3 peak of the H100 SXM
and parity of 8 device-path answers (4 small tag ORs, 4 price ranges) against the reference's distance kernel (oracle/_ref when built, else the C restatement) over
the filtered rows read back with VecSimB200_ReadRows, in (distance, docId) order.  The card name and power limit are read in the
same run.
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
from bench_int8_l2 import card  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet
POSTINGS_DOCS = 50_000_000
TAG_RANKS = range(100, 1100)
PRICE_DOCS, PRICE_LEAVES = 2_000_000, 128
K = 10
FILTER_KERNELS = ("ub_mark", "ub_popc", "ub_scan", "ub_expand", "ub_clear", "ub_fill")


def log(msg):
    print(f"[bench_hybrid_filters {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def price_leaves(np, ps, total_rows):
    """(leaves, their (min, max) value, all values sorted): docIds 5, 10, ... of the corpus, lognormal prices"""
    rng = np.random.default_rng(11)
    docs = np.arange(5, min(total_rows, 5 * PRICE_DOCS) + 1, 5, dtype=np.uint64)
    prices = np.round(rng.lognormal(4, 1, len(docs)), 2)
    extra = np.sort(rng.choice(len(docs), len(docs) // 100, replace=False))
    docs = np.concatenate([docs, docs[extra]])
    prices = np.concatenate([prices, np.round(rng.lognormal(4, 1, len(extra)), 2)])
    edges = np.quantile(prices, np.linspace(0, 1, PRICE_LEAVES + 1))[1:-1]
    leaf_of = np.searchsorted(edges, prices, side="right")
    leaves, bounds = [], []
    for leaf in range(PRICE_LEAVES):
        sel = np.nonzero(leaf_of == leaf)[0]
        sel = sel[np.argsort(docs[sel], kind="stable")]
        w = ps.IndexWriter(numeric=True)
        add = w.L.II_IndexWriter_AddNumeric
        for d, v in zip(docs[sel].tolist(), prices[sel].tolist()):
            add(w.h, d, v)
        leaves.append(ps.NumericList(w.blocks()))
        bounds.append((float(prices[sel].min()), float(prices[sel].max())))
    return leaves, bounds, np.sort(prices)


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
    torch, L, vs = env.torch, env.L, env.vs
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
    tags = {}
    for r in TAG_RANKS:
        cap = int(S.Synth_DocFreq(POSTINGS_DOCS, r) * 1.2) + 4096
        ids = torch.empty(cap, dtype=torch.int32, device=dev)
        fr = torch.empty(cap, dtype=torch.int32, device=dev)
        assert S.Synth_Postings(POSTINGS_DOCS, r, ids.data_ptr(), fr.data_ptr(), scratch.data_ptr(), d_total.data_ptr(), h_count.ctypes.data, sp) == 0
        tags[r] = ps.PostingList(P.II_PostingList_FromDevice(ids.data_ptr(), fr.data_ptr(), int(h_count[0])))
        del ids, fr
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    leaves, leaf_bounds, sorted_prices = price_leaves(np, ps, total)
    log(f"{len(tags)} tag lists and {len(leaves)} price leaves built ({time.perf_counter() - t0:.1f} s for the leaves)")

    rng = np.random.default_rng(5)
    result, parity = {}, None
    for nq in (16, 256):
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0  # stored form: normalised
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qdev.cpu().numpy())
        tag_batch = [[tags[r] for r in rng.choice(list(TAG_RANKS), int(rng.integers(4, 201)), replace=False).tolist()] for _ in range(nq)]
        price_batch = []
        for i in range(nq):
            span = len(sorted_prices) // (1000 if i % 2 == 0 else 100)
            a = int(rng.integers(0, len(sorted_prices) - span))
            lo, hi = float(sorted_prices[a]), float(sorted_prices[a + span])
            picked = [leaves[j] for j, (mn, mx) in enumerate(leaf_bounds) if mx >= lo and mn <= hi]  # the tree walk's leaves
            price_batch.append((picked, lo, hi, 1, 1))
        out_l = torch.empty((nq, K), dtype=torch.int64, device=dev)
        out_s = torch.empty((nq, K), dtype=torch.float32, device=dev)
        out_c = torch.empty(nq, dtype=torch.int32, device=dev)
        for shape, batch in (("tag", tag_batch), ("price", price_batch)):

            def device_filters(s):
                if shape == "tag":
                    return ps.union_batch_device(batch, quick_exit=True, stream=s)
                return ps.numeric_filter_batch_device(batch, stream=s)

            def host_filters():
                out = []
                for q in batch:
                    if shape == "tag":
                        rs = ps.union(q, quick_exit=True)
                        keep = None
                    else:
                        keep = [leaf.filter(q[1], q[2], q[3], q[4]) for leaf in q[0]]
                        rs = ps.union(keep, quick_exit=True)
                    m = len(rs)  # the host wait of this path
                    out.append((rs, P.II_ResultSet_DeviceDocIds(rs.h) if m else None, P.II_ResultSet_DeviceLen(rs.h), m, keep))
                return out

            def run(sets):
                rc = index.topk_filtered_batch_device(qdev, K, [r[1] for r in sets], [r[3] for r in sets], counts=[r[2] for r in sets],
                                                      out_labels=out_l, out_scores=out_s, out_counts=out_c, stream=stream)[3]
                for r in sets:
                    if r[0] is not None:
                        r[0].free_after(stream)
                return rc

            def device_path():
                return run(device_filters(stream))

            def host_path():
                return run(host_filters())

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
            # the filter kernels' device time, and the bytes they move at least
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                sets = device_filters(stream)
                stream.synchronize()
            filter_us = sum(ev.device_time_total for ev in prof.key_averages()
                            if any(k in ev.key for k in FILTER_KERNELS) and getattr(ev, "device_time_total", 0) > 0)
            hits = sum(len(x[0]) for x in sets if x[0] is not None)
            for x in sets:
                if x[0] is not None:
                    x[0].close()
            postings = sum(len(l) for q in batch for l in (q if shape == "tag" else q[0]))
            # bitmap windows: the lists of a tag OR span the whole docId range, the price leaves docIds 5 .. 5 * PRICE_DOCS; each
            # window word is cleared, counted and expanded once (12 bytes), every posting read once (its value too for price)
            window_words = nq * ((POSTINGS_DOCS if shape == "tag" else 5 * PRICE_DOCS) // 32 + 1)
            moved = postings * (4 if shape == "tag" else 12) + window_words * 12 + hits * 4
            r["filter_ms"] = filter_us / 1000.0
            r["filter_postings"] = int(postings)
            r["filter_hits"] = int(hits)
            r["filter_bytes"] = int(moved)
            r["filter_GBs"] = moved / (filter_us * 1e-6) / 1e9 if filter_us else None
            r["filter_frac_of_peak"] = r["filter_GBs"] / PEAK_GBS if r["filter_GBs"] else None
            result[f"{shape}_nq{nq}_k{K}"] = r
            log(f"{shape} nq={nq}: {r}")
            if not args.no_parity and nq == 16:
                # 4 queries per shape on the device path: ORs of 4 terms of ranks 1000..1099 (the workload's ORs are too wide to
                # read their rows back one by one), the first 4 price ranges
                if shape == "tag":
                    batch = [[tags[r] for r in rng.choice(range(1000, 1100), 4, replace=False).tolist()] for _ in range(4)]
                else:
                    batch = batch[:4]
                sets = device_filters(stream)
                rc = index.topk_filtered_batch_device(qdev[:4], K, [r[1] for r in sets], [r[3] for r in sets], counts=[r[2] for r in sets],
                                                      out_labels=out_l[:4], out_scores=out_s[:4], out_counts=out_c[:4], stream=stream)[3]
                assert rc == 0
                for x in sets:
                    x[0].free_after(stream)
                stream.synchronize()
                dl, dsc, dc = out_l.cpu().numpy(), out_s.cpu().numpy(), out_c.cpu().numpy()
                parity = parity or {}
                parity[shape] = check_parity(env, index, total, host_filters(), qh, dl, dsc, dc)
    print(json.dumps({
        "metric": "hybrid filtered-KNN batches with OR / numeric-range pre-filters on the device", "unit": "ms per batch",
        "card": card(), "corpus": {"rows": total, "dim": DIM, "dtype": "f32", "metric": "cosine", "data": "synthetic"},
        "filters": {"tag": f"ORs of 4-200 terms of ranks {TAG_RANKS.start}..{TAG_RANKS.stop - 1}, synthetic Zipf over {POSTINGS_DOCS} docs",
                    "price": f"0.1 % / 1 % ranges over {PRICE_DOCS} docs (1 % multi-value) in {PRICE_LEAVES} leaves"},
        "k": K, "steps": args.steps, "warmup": args.warmup, "peak_GBs": PEAK_GBS, "results": result, "parity": parity}))
    env.close()


def check_parity(env, index, total, host_sets, qh, dl, dsc, counts):
    """The host-built filters' docIds, their rows read back from HBM, the reference's distances, against the device path's rows."""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    L = env.L
    ids_ok, bits_ok, n_checked = True, True, 0
    for i, (rs, _, _, m, _) in enumerate(host_sets):
        if n_checked == 4:
            break
        if not 0 < m <= 200_000:
            continue
        ids = rs.fetch(want_freqs=False)[0]
        ids = ids[ids <= total]  # docIds past the corpus have no row
        rows = np.empty((len(ids), DIM), dtype=np.float32)
        for j, d in enumerate(ids.tolist()):
            assert L.VecSimB200_ReadRows(index.h, int(d) - 1, 1, rows[j].ctypes.data) == 0
        q = np.ascontiguousarray(qh[i])
        dist = np.empty(len(ids), dtype=np.float32)
        if ol.ref_vecsim() is not None:
            ol.ref_vecsim().Ref_Distances(ol.F32, ol.COS, DIM, ol._p(rows), rows.strides[0], len(ids), ol._p(q), ol._p(dist))
        else:
            for j in range(len(ids)):
                dist[j] = ol.port().orc_distance(ol.F32, ol.COS, DIM, ol._p(rows[j]), ol._p(q), ol.TIER_AVX512)
        order = np.lexsort((ids, dist))[:K]
        n = len(order)
        ids_ok &= int(counts[i]) == n and dl[i, :n].tolist() == ids[order].astype(np.int64).tolist()
        bits_ok &= dsc[i, :n].tobytes() == dist[order].tobytes()
        n_checked += 1
    for rs, *_ in host_sets:
        rs.close()
    return {"queries": n_checked, "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok),
            "checker": ("reference distance kernel (oracle/_ref)" if ol.ref_vecsim() is not None else "C restatement of the reference")
                       + " over the filtered rows read back from HBM, order (distance, docId)"}


if __name__ == "__main__":
    main()
