"""Device range-batch benchmark (VecSimB200_RangeQueryBatchDevice): prints one JSON line.

Workloads: FLAT 10M x 768 synthetic rows, 256 queries per batch, each query's radius the exact distance of its 10th and, in a
second run, its 100th nearest neighbour (one VecSimB200_TopKQueryBatchDevice with k = 100):
  fp32 cosine                 the device API against VecSimB200_RangeQueryBatch (the same fp32 route, host blobs in, replies out)
  int8 / uint8, L2 and IP     the device API (the fixed-radius pass on the integer tensor cores) against VecSimB200_RangeQueryBatch,
                              which answers these types with one exact scan per query: it is timed on the first 8 queries only and
                              reported per query
  fp16 / bf16, IP and cosine  the device API (the direct 16-bit fixed-bound pass with the margin eps16_q and CUDA-core rescoring)
                              against the same batch under VecSimB200_SetCoarseMode(0), the exact scan the route replaces (one
                              timed batch: "before"), and the host API as for 8-bit types.  The cases are opt-in (--cases).
                              Rows are ingested as generated (AddVectorsDevice normalises nothing), so the cosine cases differ
                              from the inner-product ones only in their normalised queries
Per run: ms per device batch (CUDA events around the call, median of --steps after --warmup), the main pass's device time
(VecSimB200_GetStats) against the HBM floor of reading the rows it streams once (fp32: the 15.36 GB fp16 shadow; 8-bit: 7.68 GB),
the queries each route answered (VecSimB200_LastCoarseFlags), and, at the 10th neighbour, 16 queries against the C restatement of
the reference run over the device's own rows (read back with VecSimB200_ReadRows): equal ids and score bits (fp16 / bf16: the
reference's own 16-bit arithmetic differs in the last bits, so ids equal away from the radius and scores within the 1e-2 bar of
BASELINE, and the whole batch bit-equal to the mode-0 batch instead).  The card name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, N_ROWS, SEED_QUERIES, Env, build_shard, load_peaks, usable_cores  # noqa: E402
from bench_int8_l2 import build as build_8bit  # noqa: E402
from bench_range import card  # noqa: E402


def log(msg):
    print(f"[bench_range_device {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def reference_check(env, index, rows, vtype_ol, metric_ol, q_stored, radii, got, tol=0.0):
    """16 queries: the C restatement over the stored rows, 1M rows per chunk (labels = row + 1), merged and sorted by label.
    tol > 0: ids equal except those the reference scores within tol of the radius, scores of the common ids within tol"""
    from concurrent.futures import ThreadPoolExecutor

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    # fp32 / 16-bit cosine rows are stored normalised: the reference's cosine distance is the inner-product distance of the stored row
    # and the normalised query
    metric = ol.IP if metric_ol == ol.COS else metric_ol
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
        o = np.argsort(ids, kind="stable")
        if tol > 0:
            mine = dict(zip(lab[:min(int(cnt), len(lab))].tolist(), sc[:min(int(cnt), len(lab))].tolist()))
            ref = dict(zip(ids.tolist(), scores.tolist()))
            far = {j for j, v in ref.items() if v < radii[i] - tol}
            ids_ok &= far <= set(mine) and all(v <= radii[i] + tol for v in mine.values())
            bits_ok &= all(abs(mine[j] - ref[j]) <= tol for j in set(mine) & set(ref))
            continue
        ids_ok &= int(cnt) == len(ids) and lab[:len(ids)].tolist() == ids[o].tolist()
        bits_ok &= sc[:len(ids)].astype(np.float32).tobytes() == scores[o].tobytes()
    if tol > 0:
        return {"queries": len(q_stored), "ids_equal_away_from_the_radius": bool(ids_ok), f"scores_within_{tol:g}": bool(bits_ok),
                "checker": "C restatement of the reference (AVX-512 tier) over rows read back from HBM"}
    return {"queries": len(q_stored), "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok),
            "checker": "C restatement of the reference (AVX-512 tier) over rows read back from HBM"}


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cap", type=int, default=1024)
    ap.add_argument("--cases", default="f32_cos,i8_l2,i8_ip,u8_l2,u8_ip")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L, vs, S = env.torch, env.L, env.vs, env.S
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    nq, cap = args.batch, args.cap
    hbm_gbs, hbm_src = load_peaks()
    types = {"f32": (vs.VecSimType_FLOAT32, ol.F32, 4), "i8": (vs.VecSimType_INT8, ol.I8, 1), "u8": (vs.VecSimType_UINT8, ol.U8, 1),
             "f16": (vs.VecSimType_FLOAT16, ol.F16, 2), "bf16": (vs.VecSimType_BFLOAT16, ol.BF16, 2)}
    metrics = {"cos": (vs.VecSimMetric_Cosine, ol.COS), "l2": (vs.VecSimMetric_L2, ol.L2), "ip": (vs.VecSimMetric_IP, ol.IP)}
    out = {}
    for case in args.cases.split(","):
        t, m = case.split("_")
        vtype, vtype_ol, es = types[t]
        metric, metric_ol = metrics[m]
        t0 = time.perf_counter()
        if es >= 2:
            index, _ = build_shard(env, vtype, metric, args.rows, 0)
        else:
            index = build_8bit(env, vtype, metric, args.rows, DIM)
        log(f"{case}: corpus built in {time.perf_counter() - t0:.1f} s")
        pitch = index.query_pitch()
        qraw = torch.empty((nq, DIM), dtype={4: torch.float32, 2: torch.int16, 1: torch.uint8}[es], device=env.dev)
        assert S.Synth_FillRows(qraw.data_ptr(), DIM * es, vtype, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qraw.cpu().numpy())
        if vtype_ol == ol.I8:
            qh = qh.view(np.int8)
        if es == 2:
            qh = qh.view(np.uint16)
        qst = np.zeros((nq, pitch), dtype=np.uint8)  # stored form, query_pitch() apart
        for i in range(nq):
            qst[i, :qh[i].nbytes] = qh[i].view(np.uint8)
            if metric == vs.VecSimMetric_Cosine:
                vs.normalize(qst[i], DIM, vtype)
        qd = torch.from_numpy(qst).to(env.dev)
        k_lab = torch.empty((nq, 100), dtype=torch.int64, device=env.dev)
        k_sc = torch.empty((nq, 100), dtype=torch.float32, device=env.dev)
        assert L.VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, 100, k_lab.data_ptr(), k_sc.data_ptr(), None) == 0
        torch.cuda.synchronize()
        scores100 = k_sc.cpu().numpy()
        floor_gb = args.rows * DIM * (2 if es >= 2 else 1) / 1e9
        floor_ms = floor_gb / hbm_gbs * 1000.0
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        runs = {}
        for rank in (10, 100):
            radii = np.ascontiguousarray(scores100[:, rank - 1])
            rd = torch.from_numpy(radii).to(env.dev)
            lab = torch.empty((nq, cap), dtype=torch.int64, device=env.dev)
            sc = torch.empty((nq, cap), dtype=torch.float32, device=env.dev)
            cnt = torch.empty(nq, dtype=torch.int32, device=env.dev)

            def call():
                return L.VecSimB200_RangeQueryBatchDevice(index.h, qd.data_ptr(), nq, rd.data_ptr(), cap, vs.BY_SCORE, lab.data_ptr(),
                                                          sc.data_ptr(), cnt.data_ptr(), None)

            for _ in range(max(1, args.warmup)):
                assert call() == 0
            torch.cuda.synchronize()
            index.stats(reset=True)
            times = []
            for _ in range(args.steps):
                ev0.record(torch.cuda.default_stream())  # the legacy default stream: NULL in the call above
                assert call() == 0
                ev1.record(torch.cuda.default_stream())
                ev1.synchronize()
                times.append(ev0.elapsed_time(ev1))
            st = index.stats(reset=True)
            flags = np.zeros(nq, dtype=np.uint32)
            assert L.VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq) == 0
            path = L.VecSimB200_LastBatchPath(index.h)
            counts = cnt.cpu().numpy().view(np.uint32)
            main_ms = st.scan_device_us / max(1, st.scan_launches) / 1000.0
            before = None
            if es == 2:  # the same batch on the exact scan (mode 0): one timed call, and the whole batch bit-equal to the route's
                got = (lab.cpu().numpy(), sc.cpu().numpy(), counts.copy())
                L.VecSimB200_SetCoarseMode(0)
                try:
                    ev0.record(torch.cuda.default_stream())
                    assert call() == 0
                    ev1.record(torch.cuda.default_stream())
                    ev1.synchronize()
                    before_ms = ev0.elapsed_time(ev1)
                    assert L.VecSimB200_LastBatchPath(index.h) == 0
                finally:
                    L.VecSimB200_SetCoarseMode(-1)
                want = (lab.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32))
                same = [bool(got[0][i].tobytes() == want[0][i].tobytes() and got[1][i].tobytes() == want[1][i].tobytes()
                             and got[2][i] == want[2][i]) for i in range(nq)]
                before = {"exact_scan_batch_ms": before_ms, "speedup": before_ms / float(np.median(times)),
                          "queries_bit_equal_to_mode0": int(sum(same)), "mode": "VecSimB200_SetCoarseMode(0), one timed batch"}
            # the host API: the whole batch for fp32, the first 8 queries (one exact scan each) for 8-bit types
            hq = nq if es == 4 else 8
            reps = (C.c_void_p * hq)()
            hflags = np.zeros(hq, dtype=np.uint32)
            r64 = radii[:hq].astype(np.float64)
            if (r64 >= 0).all():
                L.VecSimB200_RangeQueryBatch(index.h, qh.ctypes.data, qh.strides[0], hq, r64.ctypes.data, None, vs.BY_SCORE,
                                             C.cast(reps, C.c_void_p), hflags.ctypes.data)
                for i in range(hq):
                    L.VecSimQueryReply_Free(reps[i])
                t1 = time.perf_counter()
                assert L.VecSimB200_RangeQueryBatch(index.h, qh.ctypes.data, qh.strides[0], hq, r64.ctypes.data, None, vs.BY_SCORE,
                                                    C.cast(reps, C.c_void_p), hflags.ctypes.data) == 0
                host_ms = (time.perf_counter() - t1) * 1000.0
                for i in range(hq):
                    L.VecSimQueryReply_Free(reps[i])
                host = {"queries_timed": hq, "batch_ms": host_ms, "ms_per_query": host_ms / hq,
                        "tensor_core_share": float((hflags == 1).mean())}
            else:
                host = {"note": "negative radii: the host API refuses them"}
            runs[f"radius_at_{rank}th"] = {
                "device_batch_ms": float(np.median(times)), "device_batch_ms_min": float(min(times)),
                "device_ms_per_query": float(np.median(times)) / nq, "main_pass_ms": main_ms, "hbm_floor_ms": floor_ms,
                "main_pass_vs_floor": floor_ms / main_ms if main_ms > 0 else None, "batch_path": int(path),
                "answered_by_tensor_cores": int((flags == 1).sum()), "answered_by_exact_scan": int((flags == 0).sum()),
                "mean_hits": float(counts.mean()), "over_cap": int((counts > cap).sum()), "steps": args.steps, "host_api": host}
            if before is not None:
                runs[f"radius_at_{rank}th"]["before_exact_scan"] = before
            log(f"{case} radius at the {rank}th neighbour: {runs[f'radius_at_{rank}th']}")
            if rank == 10 and not args.no_parity:
                pick = [(i * nq) // 16 for i in range(16)]
                got = [(lab[i].cpu().numpy(), sc[i].cpu().numpy(), counts[i]) for i in pick]
                # BY_ID for the check: the sort order of the reference's reply is by label there
                assert L.VecSimB200_RangeQueryBatchDevice(index.h, qd.data_ptr(), nq, rd.data_ptr(), cap, vs.BY_ID, lab.data_ptr(),
                                                          sc.data_ptr(), cnt.data_ptr(), None) == 0
                torch.cuda.synchronize()
                got = [(lab[i].cpu().numpy(), sc[i].cpu().numpy(), counts[i]) for i in pick]
                qsel = np.ascontiguousarray(qst[pick, :qh[0].nbytes]).view(ol.NP_DTYPE[vtype_ol])
                runs["parity"] = reference_check(env, index, args.rows, vtype_ol, metric_ol, qsel, radii[pick], got,
                                                 tol=1e-2 if es == 2 else 0.0)
                log(f"{case} parity: {runs['parity']}")
        out[case] = runs
        index.close()
        del qd, k_lab, k_sc
        torch.cuda.empty_cache()
    line = {"metric": f"device range batches, FLAT {args.rows} x {DIM}, batch={nq}, cap={cap}", "unit": "ms per batch",
            "value": out[next(iter(out))]["radius_at_10th"]["device_batch_ms"], "runs": out,
            "hbm_note": f"floors at {hbm_gbs:.0f} GB/s ({hbm_src})", "card": card()}
    print(json.dumps(line))
    env.close()


if __name__ == "__main__":
    main()
