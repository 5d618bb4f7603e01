"""Filtered range batches on the device (VecSimB200_HybridRangeQueryBatchDevice, DESIGN.md §4.13): prints one JSON line.

Corpora: FLAT 10M x 768 fp32 cosine and int8 L2 (bench.py's / bench_int8_l2.py's synthetic rows, device-side ingest), docIds
1..10M.  Batches of 16 and 256 queries, each query with its own device-resident random ascending filter of 0.1 %, 1 %, 10 % or 50 %
of the docIds; each query's radius is the distance of its 10th and of its 100th FILTERED neighbour (one
VecSimB200_HybridTopKBatchDevice with k = 100).  The fractions sit on both sides of the mode choice: 0.1 % takes the gather,
10 % at 256 queries the dense route.  Per case the line reports:
  auto_ms / adhoc_ms / batches_ms   wall clock per batch to stream completion (host clock around the call and a stream
      synchronise), median over the steps, in automatic mode and with each forced policy (cases whose gather reads more than
      100 GB time 3 steps)
  route             the automatic plan's route (LastBatchPath) and LastCoarseFlags after it (count per value)
  main_pass_ms      the forced dense call's main pass (CUDA events, VecSimB200_GetStats) and its share of the HBM floor of the rows
                    it streams (fp32: the 15.36 GB fp16 shadow, int8: 7.68 GB, at 3.35 TB/s)
  lost_to_cap       queries whose whole-corpus VecSimB200_LabelRangeQueryBatchDevice answer is longer than its 4096-entry cap (the
                    caller would have to fall back to the host API for them)
  equal             the three policies' rows are equal (labels, score bits, counts)
Per corpus: the host API (VecSimIndex_RangeQuery, then the intersection with the filter) on 8 timed queries of the 1 % filter at
the 100th neighbour, and 16 queries of a 256 x 1 % batch at the 10th neighbour checked against the C restatement of the reference
over rows read back from HBM (ids and score bits).  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import DIM, SEED_QUERIES, Env, build_shard, usable_cores  # noqa: E402
from bench_hybrid_dense import make_filters  # noqa: E402
from bench_int8_l2 import build as build_8bit  # noqa: E402
from bench_range import card  # noqa: E402

HBM_PEAK = 3.35e12
N_ROWS = 10_000_000
HYBRID_ADHOC_BF, HYBRID_BATCHES = 2, 3
FRACS = {"0.1%": 0.001, "1%": 0.01, "10%": 0.1, "50%": 0.5}


def log(msg):
    print(f"[bench_range_hybrid {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def reference_parity(env, index, rows, vtype_ol, metric_ol, q_stored, radii, filters, got):
    """The C restatement of the reference over the rows read back from HBM, 1M rows per chunk (labels = row + 1); each query's
    whole-corpus range answer intersected with its filter, by label, against the device's BY_ID rows"""
    from concurrent.futures import ThreadPoolExecutor

    import numpy as np
    import oracle_lib as ol

    metric = ol.IP if metric_ol == ol.COS else metric_ol  # cosine rows are stored normalised: the inner-product distance
    hits = [([], []) for _ in range(len(q_stored))]
    chunk = 1_000_000
    host = np.empty((chunk, DIM), dtype=ol.NP_DTYPE[vtype_ol])
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert env.L.VecSimB200_ReadRows(index.h, done, n, host.ctypes.data) == 0
        p = ol.PortIndex(vtype_ol, DIM, metric, tier=ol.TIER_AVX512)
        p.add_many(host[:n], done + 1)
        with ThreadPoolExecutor(max_workers=usable_cores()) as ex:
            answers = list(ex.map(lambda i: p.range(q_stored[i], float(radii[i]), 0), range(len(q_stored))))
        for i, (ids, scores) in enumerate(answers):
            hits[i][0].append(ids)
            hits[i][1].append(scores)
        del p
        done += n
    ids_ok = bits_ok = True
    for i, (lab, sc, cnt) in enumerate(got):
        ids, scores = np.concatenate(hits[i][0]), np.concatenate(hits[i][1]).astype(np.float32)
        m = np.isin(ids, filters[i])
        ids, scores = ids[m], scores[m]
        o = np.argsort(ids, kind="stable")
        ids_ok &= int(cnt) == len(ids) and lab[: len(ids)].tolist() == ids[o].tolist()
        bits_ok &= sc[: len(ids)].tobytes() == scores[o].tobytes()
    return {"queries": len(q_stored), "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok),
            "checker": "C restatement of the reference (AVX-512 tier) over rows read back from HBM"}


def run_corpus(env, args, case):
    import numpy as np
    import oracle_lib as ol

    torch, L, vs, S = env.torch, env.L, env.vs, env.S
    n, cap = args.rows, args.cap
    if case == "f32_cos":
        vtype, vtype_ol, metric, metric_ol, es = vs.VecSimType_FLOAT32, ol.F32, vs.VecSimMetric_Cosine, ol.COS, 4
        index, _ = build_shard(env, vtype, metric, n, 0)
    else:
        vtype, vtype_ol, metric, metric_ol, es = vs.VecSimType_INT8, ol.I8, vs.VecSimMetric_L2, ol.L2, 1
        index = build_8bit(env, vtype, metric, n, DIM)
    floor_ms = n * DIM * (2 if es == 4 else 1) / HBM_PEAK * 1e3
    stream = env.stream

    def params(policy):
        if policy is None:
            return None
        p = vs.VecSimQueryParams()
        p.searchMode = policy
        return p

    out, host_api, parity = {}, None, None
    for nq in [int(x) for x in args.nq.split(",")]:
        qraw = torch.empty((nq, DIM), dtype=torch.float32 if es == 4 else torch.uint8, device=env.dev)
        assert S.Synth_FillRows(qraw.data_ptr(), DIM * es, vtype, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qraw.cpu().numpy())
        if vtype_ol == ol.I8:
            qh = qh.view(np.int8)
        qst = np.zeros((nq, index.query_pitch()), dtype=np.uint8)
        for i in range(nq):
            qst[i, : qh[i].nbytes] = qh[i].view(np.uint8)
            if metric == vs.VecSimMetric_Cosine:
                vs.normalize(qst[i], DIM, vtype)
        qd = torch.from_numpy(qst).to(env.dev)
        for fname, fr in FRACS.items():
            filt = make_filters(env, n, [fr] * nq, seed=nq * 7 + len(fname))
            ptrs, caps = [f.data_ptr() for f in filt], [int(f.numel()) for f in filt]
            gather_gb = sum(caps) * (index.query_pitch() + 8) / 1e9
            kl, ks, kc, km, rc = index.hybrid_topk_batch_device(qd, 100, ptrs, caps, stream=stream)
            assert rc == 0
            stream.synchronize()
            ks, kc = ks.cpu().numpy(), kc.cpu().numpy()
            for rank in (10, 100):
                radii = np.array([ks[i, rank - 1] if kc[i] >= rank else np.nan for i in range(nq)], dtype=np.float32)
                rd = torch.from_numpy(radii).to(env.dev)
                outs, times = {}, {}

                def call(policy, order=vs.BY_SCORE):
                    lab = torch.empty((nq, cap), dtype=torch.int64, device=env.dev)
                    sc = torch.empty((nq, cap), dtype=torch.float32, device=env.dev)
                    cn = torch.empty(nq, dtype=torch.int32, device=env.dev)
                    r = index.hybrid_range_batch_device(qd, rd, cap, ptrs, caps, order=order, params=params(policy), out_labels=lab,
                                                        out_scores=sc, out_counts=cn, stream=stream)
                    assert r[4] == 0, (policy, r[4])
                    return lab, sc, cn

                steps = args.steps if gather_gb <= 100 else 3
                main_ms = None
                for name, policy in (("auto", None), ("adhoc", HYBRID_ADHOC_BF), ("batches", HYBRID_BATCHES)):
                    for _ in range(args.warmup):
                        call(policy)
                    stream.synchronize()
                    index.stats(reset=True)
                    ts = []
                    for _ in range(steps):
                        t = time.perf_counter()
                        r = call(policy)
                        stream.synchronize()
                        ts.append((time.perf_counter() - t) * 1e3)
                    st = index.stats(reset=True)
                    if name == "batches" and st.scan_launches:
                        main_ms = st.scan_device_us / st.scan_launches / 1e3
                    times[name] = round(statistics.median(ts), 3)
                    outs[name] = [x.cpu().numpy() for x in r]
                call(None)
                stream.synchronize()
                path = L.VecSimB200_LastBatchPath(index.h)
                flags = np.zeros(nq, dtype=np.uint32)
                assert L.VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data_as(C.c_void_p), nq) == 0
                base = outs["adhoc"]
                equal = all(outs[w][0].tolist() == base[0].tolist() and outs[w][1].tobytes() == base[1].tobytes() and
                            outs[w][2].tolist() == base[2].tolist() for w in ("auto", "batches"))
                # the whole-corpus call at its largest cap
                wl = torch.empty((nq, 4096), dtype=torch.int64, device=env.dev)
                ws = torch.empty((nq, 4096), dtype=torch.float32, device=env.dev)
                wc = torch.empty(nq, dtype=torch.int32, device=env.dev)
                assert index.label_range_batch_device(qd, rd, 4096, out_labels=wl, out_scores=ws, out_counts=wc, stream=stream)[3] == 0
                stream.synchronize()
                lost = int((wc.cpu().numpy().view(np.uint32) > 4096).sum())
                key = f"nq{nq}_{fname}_r{rank}"
                out[key] = {"auto_ms": times["auto"], "adhoc_ms": times["adhoc"], "batches_ms": times["batches"],
                            "route": int(path), "flags": {str(v): int((flags == v).sum()) for v in (0, 1)},
                            "main_pass_ms": round(main_ms, 3) if main_ms else None,
                            "main_pass_share_of_floor": round(floor_ms / main_ms, 3) if main_ms else None,
                            "gather_gb": round(gather_gb, 1), "mean_hits": float(base[2].mean()), "lost_to_cap": lost,
                            "equal": bool(equal), "steps": steps}
                log(f"{case} {key}: {out[key]}")
                if nq == 16 and fname == "1%" and rank == 100 and host_api is None:
                    fh = [f.cpu().numpy().astype(np.int64) for f in filt[:8]]
                    t = time.perf_counter()
                    for i in range(8):
                        ids, _, code = index.range(qh[i], float(radii[i]))
                        np.intersect1d(ids, fh[i])
                    host_api = {"queries": 8, "ms_per_query": round((time.perf_counter() - t) * 1e3 / 8, 2)}
                    log(f"{case} host API: {host_api}")
                if nq == 256 and fname == "1%" and rank == 10 and not args.no_parity:
                    lab, sc, cn = call(None, vs.BY_ID)
                    stream.synchronize()
                    pick = [(i * nq) // 16 for i in range(16)]
                    lab, sc, cn = lab.cpu().numpy(), sc.cpu().numpy(), cn.cpu().numpy().view(np.uint32)
                    got = [(lab[i], sc[i], cn[i]) for i in pick]
                    qsel = np.ascontiguousarray(qst[pick, : qh[0].nbytes]).view(ol.NP_DTYPE[vtype_ol])
                    fsel = [filt[i].cpu().numpy().astype(np.int64) for i in pick]
                    parity = reference_parity(env, index, n, vtype_ol, metric_ol, qsel, radii[pick], fsel, got)
                    log(f"{case} parity: {parity}")
            del filt
            torch.cuda.empty_cache()
    index.close()
    torch.cuda.empty_cache()
    return {"results": out, "host_api": host_api, "parity": parity, "hbm_floor_ms": round(floor_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--nq", type=str, default="16,256")
    ap.add_argument("--cap", type=int, default=1024)
    ap.add_argument("--cases", default="f32_cos,i8_l2")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    env.L.VecSimB200_SetCoarseMode(1)
    res = {}
    for case in args.cases.split(","):
        t0 = time.perf_counter()
        res[case] = run_corpus(env, args, case)
        log(f"{case} done in {time.perf_counter() - t0:.0f} s")
    all_equal = all(v["equal"] for r in res.values() for v in r["results"].values())
    print(json.dumps({"bench": "range_hybrid", "card": card(), "corpus": {"rows": args.rows, "dim": DIM}, "cap": args.cap,
                      "cases": res, "all_equal": bool(all_equal)}))
    env.close()


if __name__ == "__main__":
    main()
