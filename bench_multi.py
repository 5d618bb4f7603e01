"""KNN batches on a multi-value index (a label owns several rows, scored by its best row; DESIGN.md §4.4): prints one JSON line.

Corpus: 10M x 768 fp32 cosine, 256 queries per batch, k = 10, in two shapes:
  images   2M labels x 5 independent synthetic rows (labels contiguous)
  chunks   200K labels x 50 rows near a per-label centre, contiguous
Per shape the line reports:
  device_batch_ms / qps   VecSimB200_TopKQueryBatchDevice, CUDA events around the call, median over the steps
  host_batch_ms           VecSimB200_TopKQueryBatch end to end (host blobs in, labels out); it answers the queries the label
                          stage cannot prove one at a time
  flags                   histogram of VecSimB200_LastCoarseFlags (1 / 2 row proof tier, 0 row exact fallback, 3 label-aware
                          exact scan)
  main_kernel_ms          device time of the scan kernels of one device-API batch (VecSimB200_GetStats, CUDA events): the row
                          stage's main pass through the label-aware exact scan
  single_topk_ms          8 single VecSimIndex_TopKQuery calls (the per-query path a multi-value batch took before)
and parity of 16 queries: the reference's kernels (or the C restatement) over the rows read back with VecSimB200_ReadRows at
k * m rows, then the first k distinct labels: ids and score bits must be equal.  The card is read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, SEED_QUERIES, SEED_ROWS, Env, usable_cores  # noqa: E402
from bench_range import card  # noqa: E402


def log(msg):
    print(f"[bench_multi {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def build(env, shape, rows):
    """Rows are generated on the device, read into host memory a chunk at a time and added with their labels."""
    import numpy as np

    vs, L, S, torch = env.vs, env.L, env.S, env.torch
    index = vs.VecSimIndex(vs.VecSimType_FLOAT32, DIM, vs.VecSimMetric_Cosine, multi=True)
    assert L.VecSimB200_Reserve(index.h, rows) == 0, "cannot reserve HBM for the corpus"
    per = 5 if shape == "images" else 50
    chunk = 1_000_000 // per * per
    buf = torch.empty((chunk, DIM), dtype=torch.float32, device=env.dev)
    t0 = time.perf_counter()
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        if shape == "images":
            assert S.Synth_FillRows(buf.data_ptr(), DIM * 4, 0, SEED_ROWS, done, n, DIM, env.sp) == 0
        else:  # centres from the synthetic generator, 50 noisy copies each
            nl = (n + per - 1) // per
            cen = torch.empty((nl, DIM), dtype=torch.float32, device=env.dev)
            assert S.Synth_FillRows(cen.data_ptr(), DIM * 4, 0, SEED_ROWS, done // per, nl, DIM, env.sp) == 0
            torch.cuda.synchronize()
            g = torch.Generator(device=env.dev).manual_seed(done)
            buf[:n] = cen.repeat_interleave(per, dim=0)[:n] + 0.05 * torch.randn((n, DIM), generator=g, device=env.dev)
        torch.cuda.synchronize()
        host = np.ascontiguousarray(buf[:n].cpu().numpy())
        labels = np.arange(done, done + n, dtype=np.uint64) // per + 1
        assert index.add_many(host, labels=labels) == n
        done += n
    del buf
    assert L.VecSimB200_Flush(index.h) == 0
    return index, per, time.perf_counter() - t0


def parity(env, index, rows, per, qh, got_labels, got_scores, k):
    """16 queries: the k*m best rows over the device's stored rows (StreamingTopK: the reference's kernels when built), then the
    first k distinct labels in (score, row) order."""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    vs = env.vs
    pick = [(i * len(qh)) // 16 for i in range(16)]
    q = np.ascontiguousarray(qh[pick]).copy()
    for x in q:
        vs.normalize(x, DIM, vs.VecSimType_FLOAT32)
    # stored rows are unit vectors: the cosine distance is the inner-product distance of the stored row and the normalised query
    st = ol.StreamingTopK(ol.F32, ol.IP, DIM, q, k * per, usable_cores())
    chunk = 1_000_000
    host = np.empty((chunk, DIM), dtype=np.float32)
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert env.L.VecSimB200_ReadRows(index.h, done, n, host.ctypes.data) == 0
        st.feed(host[:n], done + 1)
        done += n
    ids_ok = bits_ok = True
    for j, i in enumerate(pick):
        r_ids, r_sc = st.result(j)
        seen, lab, sc = set(), [], []
        for rid, s in zip(r_ids.tolist(), r_sc.tolist()):
            l = (rid - 1) // per + 1
            if l not in seen:
                seen.add(l)
                lab.append(l)
                sc.append(s)
            if len(lab) == k:
                break
        ids_ok &= got_labels[i].astype(np.int64).tolist() == lab
        bits_ok &= got_scores[i].astype(np.float32).tobytes() == np.asarray(sc, dtype=np.float32).tobytes()
    return {"queries": 16, "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok), "checker": st.kind}


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default="images,chunks")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L = env.torch, env.L
    nq, k = args.batch, args.k
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
    torch.cuda.synchronize()
    qh = np.ascontiguousarray(qdev.cpu().numpy())
    out = {}
    for shape in args.shapes.split(","):
        index, per, build_s = build(env, shape, args.rows)
        log(f"{shape}: corpus built in {build_s:.1f} s")
        if shape == "chunks":  # queries near label centres, as a chunk search would see them
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
        qs_host = np.ascontiguousarray(qd.cpu().numpy())  # raw blobs: the host API normalises them
        qn = qs_host.copy()
        for x in qn:  # the device API takes stored-form (normalised) queries
            env.vs.normalize(x, DIM, env.vs.VecSimType_FLOAT32)
        qd = torch.from_numpy(qn).to(env.dev)
        out_l = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
        sp = env.stream.cuda_stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def device_batch():
            e0.record(env.stream)
            assert L.VecSimB200_TopKQueryBatchDevice(index.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
            e1.record(env.stream)
            e1.synchronize()
            return e0.elapsed_time(e1)

        for _ in range(max(1, args.warmup)):
            device_batch()
        index.stats(reset=True)
        dev_ms = [device_batch() for _ in range(args.steps)]
        stt = index.stats(reset=True)
        flags = np.zeros(nq, dtype=np.uint32)
        fl_rc = L.VecSimB200_LastCoarseFlags(index.h, flags.ctypes.data, nq)
        path = L.VecSimB200_LastBatchPath(index.h)
        host_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            hl, hs, rc = index.topk_batch(qs_host, k)
            host_ms.append((time.perf_counter() - t0) * 1000.0)
            assert rc == 0
        same = bool((out_l.cpu().numpy().astype(np.uint64) == hl).all() and out_s.cpu().numpy().tobytes() == hs.astype(np.float32).tobytes())
        index.topk(qs_host[0], k)  # scratch of the per-query path
        single = []
        for i in range(8):
            t0 = time.perf_counter()
            _, _, code = index.topk(qs_host[i], k)
            single.append((time.perf_counter() - t0) * 1000.0)
            assert code == 0
        dm = float(np.median(dev_ms))
        res = {"labels": args.rows // per, "rows_per_label": per, "device_batch_ms": dm, "device_batch_ms_min": min(dev_ms),
               "qps": nq / (dm / 1000.0), "host_batch_ms": float(np.median(host_ms)), "device_equals_host": same,
               "batch_path": int(path), "flags": np.bincount(flags, minlength=4).tolist() if fl_rc == 0 else None,
               "main_kernel_ms": stt.scan_device_us / max(1, stt.scan_launches) / 1000.0, "single_topk_ms": float(np.median(single)),
               "single_topk_batch_equiv_ms": float(np.median(single)) * nq, "build_s": build_s}
        if not args.no_parity:
            res["parity"] = parity(env, index, args.rows, per, qs_host, hl, hs, k)
        log(f"{shape}: {res}")
        out[shape] = res
        index.close()
        torch.cuda.empty_cache()
    line = {"metric": f"multi-value KNN QPS, FLAT {args.rows} x {DIM} fp32 cosine, batch={nq}, k={k}", "unit": "queries/s",
            "value": out[next(iter(out))]["qps"], "shapes": out, "card": card()}
    print(json.dumps(line))
    env.close()


if __name__ == "__main__":
    main()
