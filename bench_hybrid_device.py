"""Batches of hybrid queries on the device end to end (DESIGN.md §4.6): prints one JSON line.

Workload: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest), filtered by 2-term ANDs over the synthetic
Zipf posting lists of bench_postings (libsynth_b200): the 16 pairs of HYBRID_TERM_PAIRS for batches of 16 queries, 256 random pairs
of term ranks 1..100 for batches of 256.  Per (queries per batch, k) with k = 10 and 1000 the line reports:
  host_path_ms    II_IntersectBatch + II_ResultSet_Len per query + VecSimB200_TopKFilteredBatch (k = 10 only: it refuses k > 128),
                  wall clock per batch, median
  device_path_ms  II_IntersectBatchDevice + VecSimB200_TopKFilteredBatchDevice + II_ResultSet_FreeAfter on one stream, wall clock
                  per batch up to the stream's completion, median
  launches        kernels the vector index launched for one batch on each path (VecSimB200_GetStats)
  gather_ms       device time of the ragged gather of one device-path batch (torch.profiler), and the filtered-row bytes it read
                  (live filter entries x 3072 B) against the 3.35 TB/s data-sheet HBM3 peak of the H100 SXM
and parity of 8 device-path answers against the reference's distance kernel (oracle/_ref when built, else the C restatement) over
the filtered rows read back with VecSimB200_ReadRows, in (distance, docId) order: equal ids and equal score bits.  The card name and
power limit are read in the same run.
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
from bench_postings import HYBRID_TERM_PAIRS  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet
KS = (10, 1000)


def log(msg):
    print(f"[bench_hybrid_device {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


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
    rng = np.random.default_rng(5)
    pairs256 = []
    while len(pairs256) < 256:
        a, b = (int(x) for x in rng.integers(1, 101, 2))
        if a != b:
            pairs256.append((min(a, b), max(a, b)))
    batches = {16: HYBRID_TERM_PAIRS, 256: pairs256}
    chunks = (total + 1023) // 1024
    scratch = torch.empty(2 * chunks + 16, dtype=torch.int32, device=dev)
    d_total = torch.zeros(4, dtype=torch.int32, device=dev)
    h_count = np.zeros(4, dtype=np.uint32)
    lists, keep = {}, []
    for r in sorted({r for pairs in batches.values() for pr in pairs for r in pr}):
        cap = int(S.Synth_DocFreq(total, r) * 1.2) + 4096
        ids = torch.empty(cap, dtype=torch.int32, device=dev)
        fr = torch.empty(cap, dtype=torch.int32, device=dev)
        assert S.Synth_Postings(total, r, ids.data_ptr(), fr.data_ptr(), scratch.data_ptr(), d_total.data_ptr(), h_count.ctypes.data, sp) == 0
        n = int(h_count[0])
        keep.append((ids, fr))
        lists[r] = ps.PostingList(P.II_PostingList_FromDevice(ids.data_ptr(), fr.data_ptr(), n))
    torch.cuda.synchronize()
    log(f"{len(lists)} posting lists built")

    result, parity = {}, None
    for nq, pairs in batches.items():
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0  # stored form: normalised
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qdev.cpu().numpy())
        batch = [[lists[a], lists[b]] for a, b in pairs]
        # host path inputs
        arrays = [(C.c_void_p * 2)(lists[a].h, lists[b].h) for a, b in pairs]
        lists_pp = (C.c_void_p * nq)(*[C.cast(x, C.c_void_p) for x in arrays])
        n_lists = (C.c_size_t * nq)(*([2] * nq))
        rs_out = (C.c_void_p * nq)()
        q_ptrs = (C.c_void_p * nq)(*[qh[i].ctypes.data for i in range(nq)])
        id_ptrs, id_counts = (C.c_void_p * nq)(), (C.c_size_t * nq)()
        for k in KS:
            out_l = torch.empty((nq, k), dtype=torch.int64, device=dev)
            out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
            out_c = torch.empty(nq, dtype=torch.int32, device=dev)

            def device_path():
                res = ps.intersect_batch_device(batch, stream=stream)
                rc = index.topk_filtered_batch_device(qdev, k, [r[1] for r in res], [r[3] for r in res], counts=[r[2] for r in res],
                                                      out_labels=out_l, out_scores=out_s, out_counts=out_c, stream=stream)[3]
                for r in res:
                    if r[0] is not None:
                        r[0].free_after(stream)
                return rc

            def host_path():
                P.II_IntersectBatch(nq, lists_pp, n_lists, rs_out)
                for i in range(nq):
                    m = P.II_ResultSet_Len(rs_out[i]) if rs_out[i] else 0
                    id_counts[i] = m
                    id_ptrs[i] = P.II_ResultSet_DeviceDocIds(rs_out[i]) if m else None
                b_l = np.zeros((nq, k), dtype=np.uint64)
                b_s = np.zeros((nq, k), dtype=np.float64)
                b_c = (C.c_size_t * nq)()
                rc = L.VecSimB200_TopKFilteredBatch(index.h, q_ptrs, nq, k, id_ptrs, id_counts, b_l.ctypes.data, b_s.ctypes.data, b_c)
                for i in range(nq):
                    if rs_out[i]:
                        P.II_ResultSet_Free(rs_out[i])
                return rc

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
                assert device_path() == 0
                if k <= 128:
                    assert host_path() == 0
            torch.cuda.synchronize()
            r = {"device_path_ms": timed(device_path)}
            index.stats(reset=True)
            assert device_path() == 0
            stream.synchronize()
            r["launches"] = {"device_path": int(index.stats(reset=True).kernel_launches)}
            if k <= 128:
                r["host_path_ms"] = timed(host_path)
                index.stats(reset=True)
                assert host_path() == 0
                r["launches"]["host_path"] = int(index.stats(reset=True).kernel_launches)
                r["speedup"] = r["host_path_ms"] / r["device_path_ms"]
            else:
                r["host_path_ms"] = None
                r["host_path_note"] = "VecSimB200_TopKFilteredBatch refuses k > 128"
            # the ragged gather's device time and the filtered-row bytes it read
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                assert device_path() == 0
                torch.cuda.synchronize()
            gather_us = sum(ev.device_time_total for ev in prof.key_averages()
                            if "gather_ragged_kernel" in ev.key and getattr(ev, "device_time_total", 0) > 0)
            counts = out_c.cpu().numpy()
            res = ps.intersect_batch_device(batch)
            live = sum(len(x[0]) for x in res if x[0] is not None)
            for x in res:
                if x[0] is not None:
                    x[0].close()
            row_bytes = live * DIM * 4
            r["gather_ms"] = gather_us / 1000.0
            r["filtered_entries"] = int(live)
            r["filtered_row_bytes"] = int(row_bytes)
            r["gather_GBs"] = row_bytes / (gather_us * 1e-6) / 1e9 if gather_us else None
            r["gather_frac_of_peak"] = (r["gather_GBs"] / PEAK_GBS) if r["gather_GBs"] else None
            result[f"nq{nq}_k{k}"] = r
            log(f"nq={nq} k={k}: {r}")
            if parity is None and nq == 16 and k == 10 and not args.no_parity:
                parity = check_parity(env, index, P, lists, pairs, qh, out_l.cpu().numpy(), out_s.cpu().numpy(), counts, k)
    print(json.dumps({
        "metric": "hybrid filtered-KNN batches on the device end to end (2-term AND pre-filter)", "unit": "ms per batch",
        "card": card(), "corpus": {"rows": total, "dim": DIM, "dtype": "f32", "metric": "cosine", "data": "synthetic"},
        "filters": {"16": "HYBRID_TERM_PAIRS", "256": "256 random pairs of term ranks 1..100", "postings": "synthetic Zipf (libsynth_b200)"},
        "steps": args.steps, "warmup": args.warmup, "peak_GBs": PEAK_GBS, "results": result, "parity": parity}))
    env.close()


def check_parity(env, index, P, lists, pairs, qh, dl, dsc, counts, k):
    """8 queries: the filter's docIds from II_Intersect, their rows read back from HBM, the reference's distances, (distance, docId)."""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    L = env.L
    pick = []
    for i, (a, b) in enumerate(pairs):
        rs = P.II_Intersect((C.c_void_p * 2)(lists[a].h, lists[b].h), 2)
        m = P.II_ResultSet_Len(rs) if rs else 0
        if 0 < m <= 20_000:
            ids = np.zeros(m, dtype=np.uint64)
            assert P.II_ResultSet_Fetch(rs, ids.ctypes.data, None, None) == 0
            pick.append((i, ids))
        if rs:
            P.II_ResultSet_Free(rs)
        if len(pick) == 8:
            break
    ids_ok, bits_ok = True, True
    for i, ids in pick:
        m = len(ids)
        rows = np.empty((m, DIM), dtype=np.float32)
        for j, d in enumerate(ids.tolist()):
            assert L.VecSimB200_ReadRows(index.h, int(d) - 1, 1, rows[j].ctypes.data) == 0
        q = np.ascontiguousarray(qh[i])
        dist = np.empty(m, dtype=np.float32)
        if ol.ref_vecsim() is not None:
            ol.ref_vecsim().Ref_Distances(ol.F32, ol.COS, DIM, ol._p(rows), rows.strides[0], m, ol._p(q), ol._p(dist))
        else:
            for j in range(m):
                dist[j] = ol.port().orc_distance(ol.F32, ol.COS, DIM, ol._p(rows[j]), ol._p(q), ol.TIER_AVX512)
        order = np.lexsort((ids, dist))[:k]
        n = len(order)
        ids_ok &= int(counts[i]) == n and dl[i, :n].tolist() == ids[order].astype(np.int64).tolist()
        bits_ok &= dsc[i, :n].tobytes() == dist[order].tobytes()
    return {"queries": len(pick), "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok),
            "checker": ("reference distance kernel (oracle/_ref)" if ol.ref_vecsim() is not None else "C restatement of the reference")
                       + " over the filtered rows read back from HBM, order (distance, docId)"}


if __name__ == "__main__":
    main()
