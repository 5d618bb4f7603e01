"""int8 / uint8 L2 KNN batch benchmark (the integer tensor-core route, coarse_wgmma_kernel kOp 4): prints one JSON line.

Workload: FLAT 10M x 768 int8 and uint8 corpora (synthetic rows, device-side ingest), L2, 256 queries per batch, k = 10 and 100.
Per (type, k) the line reports:
  device_batch_ms    one VecSimB200_TopKQueryBatchDevice call on device-resident queries (CUDA events around the call, median)
  host_batch_ms      one VecSimB200_TopKQueryBatch call, host blobs in, labels and scores out (wall clock, median)
  main_pass_ms       device time of the main pass (CUDA events, VecSimB200_GetStats) against two floors: reading the corpus
                     once from HBM (n * dim bytes at 3.35 TB/s) and the int8 tensor work (2 * n * dim * nq ops at 1,979 dense
                     Tops); the larger floor is the bound that applies
  ip_route           the same two times and the main pass on an inner-product index over the same rows (the s8 / u8 route
                     that existed before)
  exact_scan         one host batch with the tensor-core routes off (VecSimB200_SetCoarseMode(0)): the CUDA-core scan the L2
                     batches took before
and, per type, parity of 16 queries against the reference's own scan (Ref_ScanTopKChunk when oracle/_ref is built, else the C
restatement) over the device's rows read back with VecSimB200_ReadRows: equal ids and equal score bits.  The card name and power
limit are read in the same run.
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

from bench import DIM, N_ROWS, SEED_QUERIES, SEED_ROWS, Env, usable_cores  # noqa: E402

TENSOR_INT8_TOPS = 1979.0  # H100 SXM data sheet, dense int8, 700 W
HBM_GBS = 3350.0           # H100 SXM data sheet, HBM3


def log(msg):
    print(f"[bench_int8_l2 {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, mclk = [x.strip() for x in out.split(",")[:3]]
        return {"name": name, "power_limit": plim, "max_sm_clock": mclk}
    except Exception as e:  # nvidia-smi missing: the name from CUDA, the limit unknown
        import torch

        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "note": f"nvidia-smi unavailable: {e}"}


def build(env, vtype, metric, rows, dim):
    """Synthetic rows generated on the device and ingested device-to-device, labels = row + 1."""
    vs, L, S, torch = env.vs, env.L, env.S, env.torch
    index = vs.VecSimIndex(vtype, dim, metric)
    assert L.VecSimB200_Reserve(index.h, rows) == 0, "cannot reserve HBM for the corpus"
    chunk = min(rows, 1_000_000)
    buf = torch.empty((chunk, dim), dtype=torch.uint8, device=env.dev)
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert S.Synth_FillRows(buf.data_ptr(), dim, vtype, SEED_ROWS, done, n, dim, env.sp) == 0
        torch.cuda.synchronize()
        assert L.VecSimB200_AddVectorsDevice(index.h, buf.data_ptr(), n, done + 1) == n
        done += n
    del buf
    return index


def time_route(env, index, qdev, qh, k, steps, warmup):
    """(device batch ms, host batch ms, main pass ms, LastBatchPath); medians over `steps` after `warmup` calls of each API."""
    import numpy as np

    torch, L = env.torch, env.L
    nq = qh.shape[0]
    out_l = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
    out_s = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
    s = env.stream

    def dev_call():
        return L.VecSimB200_TopKQueryBatchDevice(index.h, qdev.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), env.sp)

    for _ in range(max(1, warmup)):
        assert dev_call() == 0
        assert index.topk_batch(qh, k)[2] == 0
    torch.cuda.synchronize()
    dev_ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        assert dev_call() == 0
        e1.record(s)
        e1.synchronize()
        dev_ms.append(e0.elapsed_time(e1))
    torch.cuda.synchronize()
    index.stats(reset=True)
    host_ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        labels, scores, rc = index.topk_batch(qh, k)
        host_ms.append((time.perf_counter() - t0) * 1000.0)
        assert rc == 0
    st = index.stats(reset=True)
    main_ms = st.scan_device_us / max(1, st.scan_launches) / 1000.0
    return float(np.median(dev_ms)), float(np.median(host_ms)), main_ms, L.VecSimB200_LastBatchPath(index.h), labels, scores


def reference_topk(env, index, rows, dim, vtype_ol, q_stored, ks):
    """The reference's scan (or the C restatement) over the device's stored rows, 1M rows per chunk; one StreamingTopK per k."""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    streams = {k: ol.StreamingTopK(vtype_ol, ol.L2, dim, q_stored, k, usable_cores()) for k in ks}
    chunk = 1_000_000
    host = np.empty((chunk, dim), dtype=ol.NP_DTYPE[vtype_ol])
    done = 0
    while done < rows:
        n = min(chunk, rows - done)
        assert env.L.VecSimB200_ReadRows(index.h, done, n, host.ctypes.data) == 0
        for s in streams.values():
            s.feed(host[:n], done + 1)
        done += n
    return streams, next(iter(streams.values())).kind


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=N_ROWS)
    ap.add_argument("--dim", type=int, default=DIM)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L, vs, S = env.torch, env.L, env.vs, env.S
    nq, dim, n = args.batch, args.dim, args.rows
    ks = (10, 100)
    hbm_floor_ms = n * dim / (HBM_GBS * 1e9) * 1e3
    tc_floor_ms = 2.0 * n * dim * nq / (TENSOR_INT8_TOPS * 1e12) * 1e3
    bound = "HBM" if hbm_floor_ms >= tc_floor_ms else "int8 tensor"
    floor_ms = max(hbm_floor_ms, tc_floor_ms)
    L.VecSimB200_SetCoarseMode(1)
    result = {}
    for vname, vtype, vtype_ol in (("int8", vs.VecSimType_INT8, 4), ("uint8", vs.VecSimType_UINT8, 5)):
        qdev = torch.empty((nq, dim), dtype=torch.uint8, device=env.dev)
        assert S.Synth_FillRows(qdev.data_ptr(), dim, vtype, SEED_QUERIES, 0, nq, dim, env.sp) == 0
        torch.cuda.synchronize()
        qh = np.ascontiguousarray(qdev.cpu().numpy().view(np.int8 if vtype == vs.VecSimType_INT8 else np.uint8))
        t0 = time.perf_counter()
        l2 = build(env, vtype, vs.VecSimMetric_L2, n, dim)
        log(f"{vname} L2 corpus built in {time.perf_counter() - t0:.1f} s")
        per_k = {}
        answers = {}
        for k in ks:
            dev_ms, host_ms, main_ms, path, labels, scores = time_route(env, l2, qdev, qh, k, args.steps, args.warmup)
            assert path == 2, f"the {vname} L2 batch did not take the tensor-core route (path {path})"
            answers[k] = (labels, scores)
            per_k[k] = {"device_batch_ms": dev_ms, "host_batch_ms": host_ms, "main_pass_ms": main_ms,
                        "device_qps": nq / (dev_ms / 1e3), "main_pass_share_of_hbm_floor": hbm_floor_ms / main_ms,
                        "main_pass_share_of_int8_tensor_floor": tc_floor_ms / main_ms, "last_batch_path": path}
            log(f"{vname} L2 k={k}: {per_k[k]}")
        # the CUDA-core exact scan, once per k
        L.VecSimB200_SetCoarseMode(0)
        for k in ks:
            l2.stats(reset=True)
            t0 = time.perf_counter()
            el, es, rc = l2.topk_batch(qh, k)
            wall = (time.perf_counter() - t0) * 1000.0
            st = l2.stats(reset=True)
            assert rc == 0 and L.VecSimB200_LastBatchPath(l2.h) == 0
            same = el.tobytes() == answers[k][0].tobytes() and es.astype(np.float32).tobytes() == answers[k][1].astype(np.float32).tobytes()
            per_k[k]["exact_scan"] = {"host_batch_ms": wall, "scan_ms": st.scan_device_us / max(1, st.scan_launches) / 1000.0,
                                      "same_answer": same}
            log(f"{vname} exact scan k={k}: {per_k[k]['exact_scan']}")
        L.VecSimB200_SetCoarseMode(1)
        parity = None
        if not args.no_parity:
            pick = [(i * nq) // 16 for i in range(16)]
            streams, kind = reference_topk(env, l2, n, dim, vtype_ol, np.ascontiguousarray(qh[pick]), ks)
            parity = {"queries": 16, "checker": kind}
            for k in ks:
                ids_ok = bits_ok = True
                for j, i in enumerate(pick):
                    ri, rs = streams[k].result(j)
                    ids_ok &= answers[k][0][i].astype(np.int64).tolist() == ri.tolist()
                    bits_ok &= answers[k][1][i].astype(np.float32).tobytes() == rs.astype(np.float32).tobytes()
                parity[f"k{k}"] = {"ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok)}
            parity["ok"] = all(v["ids_equal"] and v["score_bits_equal"] for v in parity.values() if isinstance(v, dict))
            log(f"{vname} parity: {parity}")
        l2.close()
        torch.cuda.empty_cache()
        # the inner-product route on the same rows, for comparison
        ip = build(env, vtype, vs.VecSimMetric_IP, n, dim)
        for k in ks:
            dev_ms, host_ms, main_ms, path, _, _ = time_route(env, ip, qdev, qh, k, args.steps, args.warmup)
            per_k[k]["ip_route"] = {"device_batch_ms": dev_ms, "host_batch_ms": host_ms, "main_pass_ms": main_ms, "last_batch_path": path}
            log(f"{vname} IP k={k}: {per_k[k]['ip_route']}")
        ip.close()
        del qdev
        torch.cuda.empty_cache()
        result[vname] = {f"k{k}": v for k, v in per_k.items()}
        result[vname]["parity"] = parity
    L.VecSimB200_SetCoarseMode(-1)
    line = {"metric": f"int8 / uint8 L2 batch QPS, FLAT {n} x {dim}, batch={nq}, k=10 (int8, device API)", "unit": "queries/s",
            "value": result["int8"]["k10"]["device_qps"], "runs": result,
            "floors": {"hbm_ms": hbm_floor_ms, "int8_tensor_ms": tc_floor_ms, "bound": bound, "floor_ms": floor_ms,
                       "note": f"{n * dim / 1e9:.2f} GB at {HBM_GBS:.0f} GB/s; {2.0 * n * dim * nq / 1e12:.2f} Tops at "
                               f"{TENSOR_INT8_TOPS:.0f} dense Tops (H100 SXM data sheet, 700 W)"},
            "card": card()}
    print(json.dumps(line))
    env.close()


if __name__ == "__main__":
    main()
