"""Range-query batch benchmark (VecSimB200_RangeQueryBatch): prints one JSON line.

Default workload: the config-2 corpus of bench.py (FLAT 10M x 768 fp32, cosine, synthetic rows), 256 queries per batch.
Each query's radius is the exact distance of its 10th nearest neighbour in one run and of its 100th in another, both
taken from one VecSimB200_TopKQueryBatch with k = 100.  Per run the line reports:
  batch_ms / range_qps      wall time of one VecSimB200_RangeQueryBatch call (host blobs in, replies out)
  main_pass_ms              device time of the fixed-bound main pass (CUDA events, VecSimB200_GetStats), against the HBM
                            floor of reading the 15.36 GB fp16 shadow once
  proven_share              share of queries answered by the tensor-core route (flag 1); the rest took one exact scan each
  mean_hits                 mean reply length
and, once: the time of single VecSimIndex_RangeQuery calls on 8 of the queries, and parity of 16 queries against the C
restatement of the reference run on the device's own rows (read back with VecSimB200_ReadRows, 1M rows at a time, merged
and sorted by (score, label)): equal ids and equal score bits.  The card name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, N_ROWS, SEED_QUERIES, Env, build_shard, load_peaks, usable_cores  # noqa: E402


def log(msg):
    print(f"[bench_range {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, mclk = [x.strip() for x in out.split(",")[:3]]
        return {"name": name, "power_limit": plim, "max_sm_clock": mclk}
    except Exception as e:  # nvidia-smi missing: the name from CUDA, the limit unknown
        import torch

        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "note": f"nvidia-smi unavailable: {e}"}


def reference_ranges(env, index, rows, q_stored, radii_sets):
    """Range answers of the C restatement over the device's stored rows, 1M rows per chunk (labels = row + 1), merged;
    one list of (ids, scores) per radius set, each sorted by (score, label)."""
    from concurrent.futures import ThreadPoolExecutor

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    # the stored rows are normalised already: the cosine distance of the reference is the inner-product distance of the
    # stored row and the normalised query, so the chunks go into an inner-product index (which stores them unchanged)
    hits = [[([], []) for _ in range(len(q_stored))] for _ in radii_sets]
    chunk = 1_000_000
    host = np.empty((chunk, DIM), dtype=np.float32)
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert env.L.VecSimB200_ReadRows(index.h, done, n, host.ctypes.data) == 0
        p = ol.PortIndex(ol.F32, DIM, ol.IP, tier=ol.TIER_AVX512)
        p.add_many(host[:n], done + 1)
        jobs = [(s, i) for s in range(len(radii_sets)) for i in range(len(q_stored))]
        with ThreadPoolExecutor(max_workers=usable_cores()) as ex:  # one query per core (ctypes releases the GIL)
            answers = list(ex.map(lambda j: p.range(q_stored[j[1]], float(radii_sets[j[0]][j[1]])), jobs))
        for (s, i), (ids, scores) in zip(jobs, answers):
            hits[s][i][0].append(ids)
            hits[s][i][1].append(scores)
        del p
        done += n
        log(f"reference ranges over rows [0, {done})")
    out = []
    for per_set in hits:
        merged = []
        for ids, scores in per_set:
            ids, scores = np.concatenate(ids), np.concatenate(scores).astype(np.float32)
            o = np.lexsort((ids, scores))
            merged.append((ids[o], scores[o]))
        out.append(merged)
    return out


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L, vs, S = env.torch, env.L, env.vs, env.S
    nq = args.batch
    index, build_s = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, args.rows, 0)
    log(f"corpus built in {build_s:.1f} s")
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
    torch.cuda.synchronize()
    qh = np.ascontiguousarray(qdev.cpu().numpy())  # raw host blobs: the library normalises them, as VecSimIndex_RangeQuery does
    del qdev

    # radii: the exact distances of the 10th and the 100th neighbour, from one top-100 batch
    labels100, scores100, rc = index.topk_batch(qh, 100)
    assert rc == 0
    hbm_gbs, hbm_src = load_peaks()
    shadow_gb = args.rows * DIM * 2 / 1e9
    floor_ms = shadow_gb / hbm_gbs * 1000.0

    reps = (C.c_void_p * nq)()
    flags = np.zeros(nq, dtype=np.uint32)

    def run_batch(radii):
        t0 = time.perf_counter()
        rc = L.VecSimB200_RangeQueryBatch(index.h, qh.ctypes.data, qh.strides[0], nq, radii.ctypes.data, None, vs.BY_SCORE,
                                          C.cast(reps, C.c_void_p), flags.ctypes.data)
        dt = time.perf_counter() - t0
        assert rc == 0, rc
        hits = [L.VecSimQueryReply_Len(reps[i]) for i in range(nq)]
        for i in range(nq):
            L.VecSimQueryReply_Free(reps[i])
        return dt, hits

    runs = {}
    radii_by = {}
    for rank in (10, 100):
        radii = np.ascontiguousarray(scores100[:, rank - 1].astype(np.float32).astype(np.float64))
        radii_by[rank] = radii
        for _ in range(max(1, args.warmup)):
            run_batch(radii)
        index.stats(reset=True)
        walls = []
        for _ in range(args.steps):
            dt, hits = run_batch(radii)
            walls.append(dt)
        st = index.stats(reset=True)
        main_ms = st.scan_device_us / max(1, st.scan_launches) / 1000.0
        batch_ms = float(np.median(walls)) * 1000.0
        runs[f"radius_at_{rank}th"] = {
            "batch_ms": batch_ms, "batch_ms_min": min(walls) * 1000.0, "range_qps": nq / (batch_ms / 1000.0),
            "main_pass_ms": main_ms, "main_pass_launches": int(st.scan_launches), "hbm_floor_ms": floor_ms,
            "main_pass_vs_floor": floor_ms / main_ms if main_ms > 0 else None,
            "proven_share": float((flags == 1).mean()), "mean_hits": float(np.mean(hits)), "steps": args.steps}
        log(f"radius at the {rank}th neighbour: {runs[f'radius_at_{rank}th']}")

    # single VecSimIndex_RangeQuery calls, for comparison (each one exact scan of the fp32 corpus)
    index.range(qh[0], float(radii_by[10][0]))  # scratch for the per-row score array
    single = []
    for i in range(8):
        t0 = time.perf_counter()
        ids, _, code = index.range(qh[i], float(radii_by[10][i]))
        single.append(time.perf_counter() - t0)
        assert code == 0
    single_ms = float(np.median(single)) * 1000.0

    parity = None
    if not args.no_parity:
        pick = [(i * nq) // 16 for i in range(16)]
        q_stored = np.ascontiguousarray(qh[pick]).copy()
        for q in q_stored:
            vs.normalize(q, DIM, vs.VecSimType_FLOAT32)
        parity = {}
        ranks = sorted(radii_by)
        refs = reference_ranges(env, index, args.rows, q_stored, [radii_by[r][pick] for r in ranks])
        for rank, ref in zip(ranks, refs):
            replies, rc, fl = index.range_batch(qh[pick], radii_by[rank][pick])
            assert rc == 0
            ids_ok = all(replies[j][0].tolist() == ref[j][0].tolist() for j in range(16))
            bits_ok = all(replies[j][1].astype(np.float32).tobytes() == ref[j][1].tobytes() for j in range(16))
            parity[f"radius_at_{rank}th"] = {"queries": 16, "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok),
                                             "proven": int((fl == 1).sum()), "hits": int(sum(len(r[0]) for r in replies))}
        parity["ok"] = all(v["ids_equal"] and v["score_bits_equal"] for v in parity.values() if isinstance(v, dict))
        parity["checker"] = "C restatement of the reference (AVX-512 tier) over rows read back from HBM"

    line = {"metric": f"range QPS, FLAT {args.rows} x {DIM} fp32 cosine, batch={nq}", "unit": "queries/s",
            "value": runs["radius_at_10th"]["range_qps"], "runs": runs,
            "single_range_query_ms": single_ms, "single_range_query_qps": 1000.0 / single_ms,
            "hbm_floor_note": f"{shadow_gb:.2f} GB fp16 shadow at {hbm_gbs:.0f} GB/s ({hbm_src})",
            "build_s": build_s, "parity": parity, "card": card()}
    print(json.dumps(line))
    index.close()
    env.close()


if __name__ == "__main__":
    main()
