"""Device range batches on a multi-value index (VecSimB200_LabelRangeQueryBatchDevice, DESIGN.md §4.12): prints one JSON line.

Corpus: bench_multi.py's, 10M x 768 fp32 cosine, in two shapes:
  images   2M labels x 5 independent synthetic rows (labels contiguous)
  chunks   200K labels x 50 rows near a per-label centre, contiguous
256 queries per batch, cap 1024, each query's radius the score of its 10th and, in a second run, its 100th LABEL neighbour (one
multi-value VecSimB200_TopKQueryBatchDevice with k = 100).  Per run:
  device_batch_ms      the device API, CUDA events around the call, median of --steps after --warmup
  main_pass_ms         the timed span of one batch (VecSimB200_GetStats): the route's main pass, or the exact scan
  flags                histogram of VecSimB200_LastCoarseFlags (1 route + fold, 3 too many hit rows to fold, 0 exact scan)
  host_api             VecSimB200_RangeQueryBatch on the first 8 queries (one exact scan per query on a multi-value index)
and, at the 10th neighbour, parity of 16 queries: the reference's own multi-value range scan (oracle/_ref) when it was built, else
the C restatement with multi=True, over the device's stored rows read back with VecSimB200_ReadRows a whole number of labels at a
time: labels, score bits and counts must be equal.  The card is read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, SEED_QUERIES, SEED_ROWS, Env, usable_cores  # noqa: E402
from bench_multi import build  # noqa: E402
from bench_range import card  # noqa: E402


def log(msg):
    print(f"[bench_range_multi {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def parity(env, index, rows, per, q_stored, radii, got):
    """Per 1M-row chunk (whole labels): a multi-value index of the chunk's stored rows, one range query per picked query; labels
    never span chunks, so the answers concatenate.  BY_ID answers compared entry for entry."""
    from concurrent.futures import ThreadPoolExecutor

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    use_ref = ol.ref_vecsim() is not None
    hits = [([], []) for _ in range(len(q_stored))]
    chunk = 1_000_000 // per * per
    host = np.empty((chunk, DIM), dtype=np.float32)
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert env.L.VecSimB200_ReadRows(index.h, done, n, host.ctypes.data) == 0
        labels = np.arange(done, done + n, dtype=np.uint64) // per + 1
        # stored rows are unit vectors: the cosine distance is the inner-product distance of the stored row and the normalised query
        if use_ref:
            ix = ol.RefIndex(ol.F32, DIM, ol.IP, multi=True)
            ix.L.Ref_AddVectors(ix.h, host.ctypes.data, n, host.strides[0], labels.ctypes.data, 0)
        else:
            ix = ol.PortIndex(ol.F32, DIM, ol.IP, multi=True, tier=ol.TIER_AVX512)
            for i in range(n):
                ix.add(host[i], int(labels[i]))
        with ThreadPoolExecutor(max_workers=usable_cores()) as ex:
            answers = list(ex.map(lambda i: ix.range(q_stored[i], float(radii[i]), 1), range(len(q_stored))))
        for i, (ids, scores) in enumerate(answers):
            hits[i][0].append(ids)
            hits[i][1].append(scores)
        del ix
        done += n
    ids_ok = bits_ok = counts_ok = True
    for i, (lab, sc, cnt) in enumerate(got):
        ids, scores = np.concatenate(hits[i][0]), np.concatenate(hits[i][1]).astype(np.float32)
        counts_ok &= int(cnt) == len(ids)
        if len(ids) <= len(lab):
            ids_ok &= lab[:len(ids)].tolist() == ids.tolist()
            bits_ok &= sc[:len(ids)].astype(np.float32).tobytes() == scores.tobytes()
    return {"queries": len(q_stored), "labels_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok), "counts_equal": bool(counts_ok),
            "checker": "reference multi-value range scan (oracle/_ref)" if use_ref else "C restatement of the reference, multi=True"}


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--cap", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default="images,chunks")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L, vs = env.torch, env.L, env.vs
    nq, cap = args.batch, args.cap
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
    torch.cuda.synchronize()
    out = {}
    for shape in args.shapes.split(","):
        index, per, build_s = build(env, shape, args.rows)
        log(f"{shape}: corpus built in {build_s:.1f} s")
        if shape == "chunks":  # queries near label centres, as bench_multi.py draws them
            g = torch.Generator(device=env.dev).manual_seed(7)
            cen = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
            pick = np.random.default_rng(7).integers(0, args.rows // per, nq)
            for i, c in enumerate(pick.tolist()):
                assert env.S.Synth_FillRows(cen[i].data_ptr(), DIM * 4, 0, SEED_ROWS, c, 1, DIM, env.sp) == 0
            torch.cuda.synchronize()
            qd = cen + 0.05 * torch.randn((nq, DIM), generator=g, device=env.dev)
        else:
            qd = qdev.clone()
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qd.cpu().numpy())  # raw blobs: the host API normalises them
        qn = qh.copy()
        for x in qn:  # the device API takes stored-form (normalised) queries
            vs.normalize(x, DIM, vs.VecSimType_FLOAT32)
        qd = torch.from_numpy(qn).to(env.dev)
        k_lab = torch.empty((nq, 100), dtype=torch.int64, device=env.dev)
        k_sc = torch.empty((nq, 100), dtype=torch.float32, device=env.dev)
        t0 = time.perf_counter()
        assert L.VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, 100, k_lab.data_ptr(), k_sc.data_ptr(), None) == 0
        torch.cuda.synchronize()
        log(f"{shape}: label neighbours in {time.perf_counter() - t0:.1f} s")
        scores100 = k_sc.cpu().numpy()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        runs = {"labels": args.rows // per, "rows_per_label": per, "build_s": build_s}
        for rank in (10, 100):
            radii = np.ascontiguousarray(scores100[:, rank - 1])
            rd = torch.from_numpy(radii).to(env.dev)
            lab = torch.empty((nq, cap), dtype=torch.int64, device=env.dev)
            sc = torch.empty((nq, cap), dtype=torch.float32, device=env.dev)
            cnt = torch.empty(nq, dtype=torch.int32, device=env.dev)

            def call(order=vs.BY_SCORE):
                return L.VecSimB200_LabelRangeQueryBatchDevice(index.h, qd.data_ptr(), nq, rd.data_ptr(), cap, order, lab.data_ptr(),
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
            # the host API: one exact scan per query on a multi-value index, timed on the first 8 queries
            hq = 8
            reps = (C.c_void_p * hq)()
            hflags = np.zeros(hq, dtype=np.uint32)
            r64 = radii[:hq].astype(np.float64)
            t1 = time.perf_counter()
            assert L.VecSimB200_RangeQueryBatch(index.h, qh.ctypes.data, qh.strides[0], hq, r64.ctypes.data, None, vs.BY_SCORE,
                                                C.cast(reps, C.c_void_p), hflags.ctypes.data) == 0
            host_ms = (time.perf_counter() - t1) * 1000.0
            same = True
            lab_h, sc_h = lab.cpu().numpy(), sc.cpu().numpy()
            for i in range(hq):
                ids, scs, _ = index._drain(reps[i])  # frees the reply
                n = len(ids)
                if n <= cap:
                    same &= int(counts[i]) == n and lab_h[i, :n].tolist() == ids.tolist() and \
                        sc_h[i, :n].tobytes() == scs.astype(np.float32).tobytes()
            res = {"device_batch_ms": float(np.median(times)), "device_batch_ms_min": float(min(times)),
                   "device_ms_per_query": float(np.median(times)) / nq,
                   "main_pass_ms": st.scan_device_us / max(1, st.scan_launches) / 1000.0, "batch_path": int(path),
                   "flags": {str(f): int((flags == f).sum()) for f in (1, 3, 0)}, "mean_labels": float(counts.mean()),
                   "over_cap": int((counts > cap).sum()), "steps": args.steps,
                   "host_api": {"queries_timed": hq, "ms_per_query": host_ms / hq, "equals_device": bool(same)}}
            log(f"{shape} radius at the {rank}th label: {res}")
            if rank == 10 and not args.no_parity:
                pick = [(i * nq) // 16 for i in range(16)]
                assert call(vs.BY_ID) == 0  # the reference's reply order by label
                torch.cuda.synchronize()
                got = [(lab[i].cpu().numpy(), sc[i].cpu().numpy(), counts[i]) for i in pick]
                res["parity"] = parity(env, index, args.rows, per, np.ascontiguousarray(qn[pick]), radii[pick], got)
                log(f"{shape} parity: {res['parity']}")
            runs[f"radius_at_{rank}th"] = res
        out[shape] = runs
        index.close()
        del qd, k_lab, k_sc
        torch.cuda.empty_cache()
    first = out[next(iter(out))]["radius_at_10th"]
    line = {"metric": f"multi-value device range batches, FLAT {args.rows} x {DIM} fp32 cosine, batch={nq}, cap={cap}",
            "unit": "ms per batch", "value": first["device_batch_ms"], "shapes": out, "card": card()}
    print(json.dumps(line))
    env.close()


if __name__ == "__main__":
    main()
