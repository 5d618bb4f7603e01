"""Filtered KNN on a multi-value index (hybrid ad-hoc queries; DESIGN.md §4.4): prints one JSON line.

Corpus: the 10M x 768 fp32 cosine multi-value corpora of bench_multi.py ("images": 2M labels x 5 rows, "chunks": 200K labels x
50 rows).  256 queries, each with its own device-resident ascending filter of about 1 % and 10 % of the labels (a random subset),
answered with one VecSimB200_TopKFilteredBatch call, k = 10.  Per shape and filter fraction the line reports:
  batch_ms           the call, host clock around it (it returns after its device work), median over the steps
  rows / bytes       rows gathered per batch (every filtered label's rows) and rows x 3,072 bytes
  gather_kernel_ms   device time covered by gather_min_kernel in one batch: the union of its launches' intervals in a
                     torch.profiler trace (the launches of different queries overlap), taken in a separate, profiled call
  hbm_fraction       bytes / gather_kernel_ms over the 3.35 TB/s data-sheet HBM3 bandwidth
  adhoc_ms_per_query what a caller can do without this path: VecSimIndex_AdhocBfCtx_GetExactDistances over the filter plus a host
                     top-k, median over 16 of the same queries (adhoc_batch_equiv_ms = that x 256)
and parity of 16 queries of the 1 % batch: the reference's getDistanceFrom fold (oracle/_ref when built, else the C restatement)
over the filtered labels' stored rows, then its ad-hoc loop: ids and score bits must be equal.  The card is read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import DIM, SEED_QUERIES, Env  # noqa: E402
from bench_multi import build  # noqa: E402
from bench_range import card  # noqa: E402

HBM_PEAK = 3.35e12


def log(msg):
    print(f"[bench_hybrid_multi {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def make_filters(env, n_labels, nq, frac, seed):
    """nq ascending uint32 docId lists on the device, each a random subset of about frac of the labels 1..n_labels."""
    torch = env.torch
    g = torch.Generator(device=env.dev).manual_seed(seed)
    out = []
    for _ in range(nq):
        keep = torch.rand(n_labels, generator=g, device=env.dev) < frac
        out.append((torch.nonzero(keep).flatten() + 1).to(torch.int32).contiguous())  # ascending; int32 holds uint32 < 2^31
    torch.cuda.synchronize()
    return out


def gather_union_ms(prof):
    spans = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                   if e.device_type.name == "CUDA" and "gather_min_kernel" in e.name)
    if not spans:
        return None
    total, cs, ce = 0.0, spans[0][0], spans[0][1]
    for s, e in spans[1:]:
        if s > ce:
            total += ce - cs
            cs, ce = s, e
        else:
            ce = max(ce, e)
    return (total + ce - cs) / 1000.0  # us -> ms


def parity(env, index, per, qs, filters, got_l, got_s, got_c, k, picks):
    """The reference's getDistanceFrom over each checked query's filtered labels: an oracle index holds exactly those labels'
    stored rows (the corpus' labels own the contiguous rows [(l-1)*per, l*per)), in row order."""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol

    torch, vs = env.torch, env.vs
    pitch, nrows = C.c_size_t(0), C.c_size_t(0)
    ptr = env.L.VecSimB200_DeviceRows(index.h, C.byref(pitch), C.byref(nrows))
    assert ptr and pitch.value % 4 == 0

    class _Rows:  # the index's HBM rows as a torch view, only read here
        __cuda_array_interface__ = {"shape": (nrows.value, pitch.value // 4), "typestr": "<f4", "data": (ptr, False), "version": 3}

    rows = torch.as_tensor(_Rows(), device=env.dev)
    kind = "reference" if ol.ref_vecsim() is not None else "port"
    ids_ok = bits_ok = True
    for i in picks:
        labs = filters[i].to(torch.int64)
        ridx = ((labs - 1)[:, None] * per + torch.arange(per, device=env.dev)[None, :]).flatten()
        host = np.ascontiguousarray(rows.index_select(0, ridx)[:, :DIM].cpu().numpy())
        # stored rows are unit vectors: the cosine distance is the inner-product distance of the stored row and the normalised query
        o = ol.RefIndex(ol.F32, DIM, ol.IP, multi=True) if kind == "reference" else ol.PortIndex(ol.F32, DIM, ol.IP, multi=True)
        hl = np.repeat(labs.cpu().numpy().astype(np.uint64), per)
        for r, lab in zip(host, hl.tolist()):
            o.add(r, lab)
        q = np.ascontiguousarray(qs[i]).copy()
        vs.normalize(q, DIM, vs.VecSimType_FLOAT32)
        best = []
        for d in labs.cpu().numpy().tolist():  # hybrid_reader.c:289-335: ascending docIds, NaN skipped, k smallest by (score, docId)
            s = o.distance_from(int(d), q)
            if s == s:
                best.append((np.float32(s), int(d)))
        best.sort()
        best = best[:k]
        c = int(got_c[i])
        ids_ok &= got_l[i, :c].astype(np.int64).tolist() == [d for _, d in best]
        bits_ok &= got_s[i, :c].astype(np.float32).tobytes() == np.array([s for s, _ in best], dtype=np.float32).tobytes()
        del o
    return {"queries": len(picks), "ids_equal": bool(ids_ok), "score_bits_equal": bool(bits_ok), "checker": kind}


def main():
    import numpy as np

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default="images,chunks")
    ap.add_argument("--fracs", default="0.01,0.1")
    ap.add_argument("--adhoc-queries", type=int, default=16)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()

    env = Env()  # refuses to run without a CUDA device
    torch, L = env.torch, env.L
    nq, k = args.batch, args.k
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, SEED_QUERIES, 0, nq, DIM, env.sp) == 0
    torch.cuda.synchronize()
    qs = np.ascontiguousarray(qdev.cpu().numpy())  # raw blobs: the library normalises them
    q_ptrs = (C.c_void_p * nq)(*[qs[i].ctypes.data for i in range(nq)])
    out = {}
    for shape in args.shapes.split(","):
        index, per, build_s = build(env, shape, args.rows)
        n_labels = args.rows // per
        log(f"{shape}: corpus built in {build_s:.1f} s")
        res_shape = {"labels": n_labels, "rows_per_label": per, "build_s": build_s}
        for fi, frac in enumerate(float(f) for f in args.fracs.split(",")):
            filters = make_filters(env, n_labels, nq, frac, 100 + fi)
            id_ptrs = (C.c_void_p * nq)(*[f.data_ptr() for f in filters])
            counts = (C.c_size_t * nq)(*[int(f.numel()) for f in filters])
            n_rows = sum(counts) * per
            out_l = np.zeros((nq, k), dtype=np.uint64)
            out_s = np.zeros((nq, k), dtype=np.float64)
            out_c = (C.c_size_t * nq)()

            def batch():
                t0 = time.perf_counter()
                assert L.VecSimB200_TopKFilteredBatch(index.h, q_ptrs, nq, k, id_ptrs, counts, out_l.ctypes.data, out_s.ctypes.data,
                                                      out_c) == 0
                return (time.perf_counter() - t0) * 1000.0

            for _ in range(max(1, args.warmup)):
                batch()
            ms = [batch() for _ in range(args.steps)]
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                batch()
            kern_ms = gather_union_ms(prof)
            # what a caller can do today: exact distances of every filtered docId through an ad-hoc context, then a host top-k
            hq = min(args.adhoc_queries, nq)
            host_f = [filters[i].cpu().numpy().astype(np.uint64) for i in range(hq)]
            index.adhoc_distances(qs[0], host_f[0][:16])  # scratch of the ad-hoc context
            adhoc_ms, adhoc_same = [], True
            for i in range(hq):
                t0 = time.perf_counter()
                d = index.adhoc_distances(qs[i], host_f[i]).astype(np.float32)
                ok = ~np.isnan(d)
                sel = np.lexsort((host_f[i][ok], d[ok]))[:k]
                top_l, top_s = host_f[i][ok][sel], d[ok][sel]
                adhoc_ms.append((time.perf_counter() - t0) * 1000.0)
                c = int(out_c[i])
                adhoc_same &= out_l[i, :c].tolist() == top_l.tolist() and out_s[i, :c].astype(np.float32).tobytes() == top_s.tobytes()
            bytes_ = n_rows * DIM * 4
            bm = float(np.median(ms))
            r = {"filter_fraction": frac, "mean_filter_labels": sum(counts) / nq, "batch_ms": bm, "batch_ms_min": min(ms),
                 "qps": nq / (bm / 1000.0), "rows": n_rows, "bytes": bytes_, "gather_kernel_ms": kern_ms,
                 "hbm_fraction": (bytes_ / (kern_ms / 1000.0)) / HBM_PEAK if kern_ms else None,
                 "batch_hbm_fraction": (bytes_ / (bm / 1000.0)) / HBM_PEAK,
                 "adhoc_ms_per_query": float(np.median(adhoc_ms)), "adhoc_batch_equiv_ms": float(np.median(adhoc_ms)) * nq,
                 "adhoc_equals_batch": bool(adhoc_same)}
            if not args.no_parity and fi == 0:
                picks = [(i * nq) // 16 for i in range(16)]
                r["parity"] = parity(env, index, per, qs, filters, out_l, out_s, out_c, k, picks)
            log(f"{shape} {frac}: {r}")
            res_shape[f"filter_{frac:g}"] = r
            del filters
        out[shape] = res_shape
        index.close()
        torch.cuda.empty_cache()
    first = out[next(iter(out))]
    line = {"metric": f"filtered KNN on a multi-value index, FLAT {args.rows} x {DIM} fp32 cosine, batch={nq}, k={k}",
            "unit": "queries/s", "value": first[next(x for x in first if x.startswith("filter_"))]["qps"], "shapes": out, "card": card()}
    print(json.dumps(line))
    env.close()


if __name__ == "__main__":
    main()
