"""KNN batches with 128 < k <= 1024 (DESIGN.md §4.5): prints one JSON line.

Workload: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest), 256 queries per batch, k = 100, 256 and
1000.  Per k the line reports:
  device_batch_ms    one VecSimB200_TopKQueryBatchDevice call on device-resident queries (CUDA events around the call, median)
  host_batch_ms      one VecSimB200_TopKQueryBatch call, host blobs in, labels and scores out (wall clock, median)
  kernels_ms         device time per kernel family of one device call, from torch.profiler (a call of its own): the sample
                     pass (adaptive_pass at k > 128, which also holds the second tier), the main pass, refine (both tiers),
                     and the exact fallback's scan and chunk selects
  flags              histogram of the per-query flags (1 = first tier, 2 = second tier, 0 = exact fallback)
  one_at_a_time      the same batch answered by VecSimIndex_TopKQuery one query at a time (wall clock), measured in this run,
                     and whether its answers equal the host batch's
and parity of the device API's answers to 16 queries per k against the reference's own scan (Ref_ScanTopKChunk when oracle/_ref is built, else the C
restatement) over the device's rows read back with VecSimB200_ReadRows: equal ids and equal score bits.  The card name and power
limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, N_ROWS, SEED_QUERIES, Env, build_shard, usable_cores  # noqa: E402
from bench_int8_l2 import card  # noqa: E402

KS = (100, 256, 1000)


def log(msg):
    print(f"[bench_large_k {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def kernel_family(name):
    if "coarse_wgmma_kernel<false, 3, 0, 2" in name:
        return "sample_pass"  # k <= 128: slice minima
    if "coarse_wgmma_kernel<false, 8, 0, 0" in name:
        return "adaptive_pass"  # k > 128: the sample pass (every stride-th tile); any k: the second tier
    if "coarse_wgmma_kernel<false, 8, 0, 1" in name or "coarse_wgmma_kernel<false, 3, 0, 1" in name:
        return "main_pass"
    if "refine_kernel" in name:
        return "refine"
    if "scan_scores_wide" in name or "scan_topk" in name:
        return "fallback_scan"
    if "select_scores_wide" in name or "final_select_wide" in name:
        return "fallback_select"
    return "other"


def profile_call(env, call):
    """Device time per kernel family of one call (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert call() == 0
        env.torch.cuda.synchronize()
    fam = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "CUDA" in str(ev.device_type) and getattr(ev, "device_time_total", 0) > 0:
            f = kernel_family(ev.key)
            fam[f] = fam.get(f, 0.0) + ev.device_time_total / 1000.0
    return fam


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--one-at-a-time", type=int, default=256, help="queries answered one at a time per k (0 = skip)")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L, vs, S = env.torch, env.L, env.vs, env.S
    nq, dim, n = args.batch, DIM, args.rows
    L.VecSimB200_SetCoarseMode(1)
    t0 = time.perf_counter()
    index, _ = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, n, 0)
    log(f"corpus built in {time.perf_counter() - t0:.1f} s")
    qdev = torch.empty((nq, dim), dtype=torch.float32, device=env.dev)
    assert S.Synth_FillRows(qdev.data_ptr(), dim * 4, 0, SEED_QUERIES, 0, nq, dim, env.sp) == 0
    assert S.Synth_NormalizeRowsF32(qdev.data_ptr(), dim * 4, nq, dim, env.sp) == 0
    torch.cuda.synchronize()
    qh = np.ascontiguousarray(qdev.cpu().numpy())
    result = {}
    answers = {}
    for k in KS:
        out_l = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=env.dev)

        def dev_call():
            return L.VecSimB200_TopKQueryBatchDevice(index.h, qdev.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), env.sp)

        for _ in range(max(1, args.warmup)):
            assert dev_call() == 0
            assert index.topk_batch(qh, k)[2] == 0
        torch.cuda.synchronize()
        dev_ms = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(env.stream)
            assert dev_call() == 0
            e1.record(env.stream)
            e1.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
        flags = np.zeros(nq, dtype=np.uint32)
        frc = L.VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)
        path = L.VecSimB200_LastBatchPath(index.h)
        dl, ds = out_l.cpu().numpy(), out_s.cpu().numpy()
        host_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            labels, scores, rc = index.topk_batch(qh, k)
            host_ms.append((time.perf_counter() - t0) * 1000.0)
            assert rc == 0
        answers[k] = (dl, ds)  # the stored-form queries the reference scans below (the host API normalises its blobs again)
        kern = profile_call(env, dev_call)
        r = {"device_batch_ms": float(np.median(dev_ms)), "host_batch_ms": float(np.median(host_ms)),
             "device_qps": nq / (float(np.median(dev_ms)) / 1e3), "last_batch_path": path, "kernels_ms": kern,
             "flags": {str(f): int((flags == f).sum()) for f in (0, 1, 2)} if frc == 0 else None}
        if args.one_at_a_time:
            m = min(nq, args.one_at_a_time)
            t0 = time.perf_counter()
            same = True
            for i in range(m):
                ids, sc, code = index.topk(qh[i], k)
                same &= code == 0 and ids.tolist() == labels[i].astype(np.int64).tolist() and \
                    sc.astype(np.float32).tobytes() == scores[i].astype(np.float32).tobytes()
            wall = (time.perf_counter() - t0) * 1000.0
            r["one_at_a_time"] = {"queries": m, "ms": wall, "ms_per_batch": wall * nq / m, "same_answers": bool(same),
                                  "speedup_of_host_batch": wall * nq / m / r["host_batch_ms"]}
        result[f"k{k}"] = r
        log(f"k={k}: {r}")
    L.VecSimB200_SetCoarseMode(-1)
    parity = None
    if not args.no_parity:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_lib as ol

        pick = [(i * nq) // 16 for i in range(16)]
        streams = {k: ol.StreamingTopK(ol.F32, ol.COS, dim, np.ascontiguousarray(qh[pick]), k, usable_cores()) for k in KS}
        chunk = 1_000_000
        host = np.empty((chunk, dim), dtype=np.float32)
        done = 0
        while done < n:
            m = min(chunk, n - done)
            assert L.VecSimB200_ReadRows(index.h, done, m, host.ctypes.data) == 0
            for s in streams.values():
                s.feed(host[:m], done + 1)
            done += m
        parity = {"queries": 16, "checker": next(iter(streams.values())).kind}
        for k in KS:
            ids_ok = bits_ok = True
            for j, i in enumerate(pick):
                ri, rs = streams[k].result(j)
                ids_ok &= answers[k][0][i].tolist() == ri.tolist()
                bits_ok &= answers[k][1][i].tobytes() == rs.astype(np.float32).tobytes()
            parity[f"k{k}"] = {"ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok)}
        parity["ok"] = all(v["ids_equal"] and v["score_bits_equal"] for v in parity.values() if isinstance(v, dict))
        log(f"parity: {parity}")
    line = {"metric": f"fp32 cosine KNN batch QPS, FLAT {n} x {dim}, batch={nq}, k=1000 (device API)", "unit": "queries/s",
            "value": result["k1000"]["device_qps"], "runs": result, "parity": parity, "card": card()}
    print(json.dumps(line))
    index.close()
    env.close()


if __name__ == "__main__":
    main()
