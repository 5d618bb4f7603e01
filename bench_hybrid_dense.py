"""Hybrid KNN batches on two device routes (VecSimB200_HybridTopKBatchDevice, DESIGN.md §4.10): prints one JSON line.

Corpus: FLAT 10M x 768 fp32 cosine (bench.py's synthetic corpus, device-side ingest), docIds 1..10M.  Batches of 16 and 256
queries, k = 10 and 1000, each query with its own device-resident random ascending filter of 0.1 %, 1 %, 10 % or 50 % of the
labels, and a mixed batch (half 0.1 %, half 10 %).  The fractions sit on both sides of the mode choice: 0.1 % takes the gather,
10 % and 50 % the dense route, 1 % is near the boundary.  Per shape the line reports:
  filtered_ms / auto_ms / adhoc_ms / batches_ms   wall clock per batch to stream completion (host clock around the call and a
      stream synchronise), median over the steps, for VecSimB200_TopKFilteredBatchDevice, the new call in automatic mode and with
      each forced policy (shapes whose gather reads more than 100 GB time 3 steps)
  modes / flags     the routes the automatic plan chose (count per route) and LastCoarseFlags after it (count per value)
  equal             every row of every timed variant equals TopKFilteredBatchDevice's: labels, score bits, counts
  ref_ok            8 queries: each answer row read back with VecSimB200_ReadRows and scored by the reference's distance
                    (oracle/_ref when built, else the C restatement): ids = the filtered call's, score bits equal
The profile (a run of its own, torch.profiler, one dense batch of 256 queries at 10 %, k = 10) gives the main pass's and the
bitmap build's kernel times and the main pass against the shadow's HBM floor (15.36 GB / 3.35 TB/s).  The card's name, power
limit and max SM clock are read in the same run.
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

from bench import DIM, SEED_QUERIES, Env, build_shard  # noqa: E402
from bench_range import card  # noqa: E402

HBM_PEAK = 3.35e12
N_ROWS = 10_000_000
EMPTY_MODE, HYBRID_ADHOC_BF, HYBRID_BATCHES = 0, 2, 3


def log(msg):
    print(f"[bench_hybrid_dense {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def make_filters(env, n_labels, fracs, seed):
    """One ascending int32 docId tensor per query: a random subset of about fracs[i] of the labels 1..n_labels."""
    torch = env.torch
    g = torch.Generator(device=env.dev).manual_seed(seed)
    out = []
    for f in fracs:
        keep = torch.rand(n_labels, generator=g, device=env.dev) < f
        out.append((torch.nonzero(keep).flatten() + 1).to(torch.int32).contiguous())
    torch.cuda.synchronize()
    return out


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--nq", type=str, default="16,256")
    ap.add_argument("--k", type=str, default="10,1000")
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()

    env = Env()
    torch, L, vs = env.torch, env.L, env.vs
    L.VecSimB200_SetCoarseMode(1)
    n = args.rows
    t0 = time.perf_counter()
    index, _ = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, n, 0)
    log(f"corpus built in {time.perf_counter() - t0:.1f} s")
    stream = env.stream
    shapes = {"0.1%": [0.001], "1%": [0.01], "10%": [0.1], "50%": [0.5], "mixed": [0.001, 0.1]}
    result, ref_ok = {}, True
    import oracle_lib as ol

    def params(policy):
        if policy is None:
            return None
        p = vs.VecSimQueryParams()
        p.searchMode = policy
        return p

    for nq in [int(x) for x in args.nq.split(",")]:
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, env.sp) == 0
        torch.cuda.synchronize()
        qh = qdev.cpu().numpy()
        for name, fr in shapes.items():
            fracs = [fr[i * len(fr) // nq] for i in range(nq)]
            filt = make_filters(env, n, fracs, seed=nq * 7 + len(name))
            ptrs = [f.data_ptr() for f in filt]
            caps = [int(f.numel()) for f in filt]
            gather_gb = sum(caps) * DIM * 4 / 1e9
            for k in [int(x) for x in args.k.split(",")]:
                outs = {}

                def call(which):
                    lab = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
                    sc = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
                    cn = torch.empty(nq, dtype=torch.int32, device=env.dev)
                    modes = None
                    if which == "filtered":
                        rc = index.topk_filtered_batch_device(qdev, k, ptrs, caps, out_labels=lab, out_scores=sc, out_counts=cn, stream=stream)[3]
                    else:
                        pol = {"auto": None, "adhoc": HYBRID_ADHOC_BF, "batches": HYBRID_BATCHES}[which]
                        r = index.hybrid_topk_batch_device(qdev, k, ptrs, caps, params=params(pol), out_labels=lab, out_scores=sc, out_counts=cn,
                                                           stream=stream)
                        rc, modes = r[4], r[3]
                    assert rc == 0, (which, rc)
                    return lab, sc, cn, modes

                steps = args.steps if gather_gb <= 100 else 3
                times = {}
                for which in ("filtered", "auto", "adhoc", "batches"):
                    for _ in range(args.warmup):
                        call(which)
                    stream.synchronize()
                    ts = []
                    for _ in range(steps):
                        t = time.perf_counter()
                        r = call(which)
                        stream.synchronize()
                        ts.append((time.perf_counter() - t) * 1e3)
                    times[which] = round(statistics.median(ts), 3)
                    outs[which] = r
                # flags of the automatic plan: one more call, then the flags
                lab, sc, cn, modes = call("auto")
                stream.synchronize()
                flags = np.zeros(nq, dtype=np.uint32)
                assert L.VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data_as(C.c_void_p), nq) == 0
                base = [x.cpu().numpy() for x in outs["filtered"][:3]]
                equal = True
                for which in ("auto", "adhoc", "batches"):
                    got = [x.cpu().numpy() for x in outs[which][:3]]
                    equal &= got[0].tolist() == base[0].tolist() and got[1].tobytes() == base[1].tobytes() and got[2].tolist() == base[2].tolist()
                ok = check_reference(ol, index, qh, base, k, [0, 1, 2, 3, nq - 4, nq - 3, nq - 2, nq - 1])
                ref_ok &= ok
                key = f"nq{nq}_k{k}_{name}"
                result[key] = {
                    "filtered_ms": times["filtered"], "auto_ms": times["auto"], "adhoc_ms": times["adhoc"], "batches_ms": times["batches"],
                    "speedup_auto_vs_filtered": round(times["filtered"] / times["auto"], 2), "gather_gb": round(gather_gb, 1),
                    "modes": {"adhoc": int((modes == HYBRID_ADHOC_BF).sum()), "batches": int((modes == HYBRID_BATCHES).sum())},
                    "flags": {str(v): int((flags == v).sum()) for v in (0, 1, 2)}, "equal": bool(equal), "ref_ok": bool(ok), "steps": steps,
                }
                log(f"{key}: {result[key]}")
            del filt
            torch.cuda.empty_cache()
    prof = None if args.no_profile else profile(env, index, n)
    print(json.dumps({"bench": "hybrid_dense", "card": card(), "corpus": {"rows": n, "dim": DIM, "dtype": "f32", "metric": "cosine"},
                      "results": result, "profile": prof, "all_equal": all(v["equal"] for v in result.values()), "ref_ok": bool(ref_ok)}))


def check_reference(ol, index, qh, base, k, qids):
    """Each answer row of the listed queries, read back from the device, scored by the reference: score bits equal.  Cosine rows
    and queries are stored normalised, so the reference's inner-product distance over them is the cosine distance."""
    import numpy as np

    lab, sc, cn = base
    ok = True
    for q in qids:
        c = int(cn[q])
        if c == 0:
            continue
        o = ol.RefIndex(ol.F32, DIM, ol.IP) if ol.ref_vecsim() is not None else ol.PortIndex(ol.F32, DIM, ol.IP, tier=ol.TIER_AVX512)
        rows = np.empty((c, DIM), dtype=np.float32)
        for j in range(c):  # labels = row + 1 (no deletes)
            assert index.L.VecSimB200_ReadRows(index.h, int(lab[q, j]) - 1, 1, rows[j:].ctypes.data_as(C.c_void_p)) == 0
        o.add_many(rows, 0)
        d = np.array([np.float32(o.distance_from(j, qh[q])) for j in range(c)], dtype=np.float32)
        ok &= d.tobytes() == sc[q, :c].tobytes()
        key = list(zip(sc[q, :c].tolist(), lab[q, :c].tolist()))
        ok &= key == sorted(key)
    return ok


def profile(env, index, n):
    """Kernel times of one dense batch (256 queries, 10 %, k = 10) from torch.profiler, in a run of its own."""
    torch = env.torch
    nq, k = 256, 10
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
    assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, env.sp) == 0
    filt = make_filters(env, n, [0.1] * nq, seed=99)
    ptrs, caps = [f.data_ptr() for f in filt], [int(f.numel()) for f in filt]
    p = env.vs.VecSimQueryParams()
    p.searchMode = HYBRID_BATCHES
    for _ in range(2):
        index.hybrid_topk_batch_device(qdev, k, ptrs, caps, params=p, stream=env.stream)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile as tprof

    with tprof(activities=[ProfilerActivity.CUDA]) as pr:
        for _ in range(3):
            index.hybrid_topk_batch_device(qdev, k, ptrs, caps, params=p, stream=env.stream)
        torch.cuda.synchronize()
    ev = [e for e in pr.events() if e.device_type.name == "CUDA"]

    def per_call(pred):
        ds = [e.time_range.end - e.time_range.start for e in ev if pred(e.name)]
        return round(sum(ds) / 3 / 1e3, 3) if ds else None  # us -> ms per batch

    main_ms = None
    coarse = sorted((e.time_range.end - e.time_range.start for e in ev if "coarse_wgmma_kernel" in e.name), reverse=True)
    if coarse:
        main_ms = round(statistics.median(coarse[:3]) / 1e3, 3)  # the main pass: the longest coarse launch of each batch
    shadow_bytes = n * ((DIM * 2 + 255) // 256 * 256)
    return {"batch": "256 queries, 10 %, k = 10, HYBRID_BATCHES", "main_pass_ms": main_ms,
            "main_pass_hbm_floor_ms": round(shadow_bytes / HBM_PEAK * 1e3, 3),
            "main_pass_share_of_floor": round(shadow_bytes / HBM_PEAK * 1e3 / main_ms, 3) if main_ms else None,
            "bitmap_build_ms": per_call(lambda s: "filter_bitmap_kernel" in s),
            "sample_and_refine_ms": per_call(lambda s: "refine_kernel" in s or "threshold_kernel" in s),
            "gather_ms": per_call(lambda s: "gather_ragged_kernel" in s)}


if __name__ == "__main__":
    main()
