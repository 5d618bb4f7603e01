#!/usr/bin/env python3
"""Sharded filtered KNN and range batches (DESIGN.md §6.1): the list merge, and the collectives against the paths they replace.

  (a) VecSimB200_MergeShardListBlocks alone on synthetic blocks: G in {2, 4, 8}, nq = 256, top-w at w in {10, 1000} (full runs),
      range at w in {1024, 4096} (runs adding up to exactly w).  Kernel time from CUDA events over many launches; the bytes of
      the runs read once and the rows written, against the HBM floor.
  (b) The config-5 step (10M x 768 fp32 cosine, a 2-term AND per query, k = 10, 16 and 256 queries): the host path of
      bench_postings.run_config5 (II_IntersectBatch -> TopKFilteredBatch -> a host-packed block -> torch all-gather ->
      MergeShardBlocks) against II_IntersectBatchDevice -> VecSimB200_ShardGroup_HybridTopKBatchDevice with no host wait.
  (c) VecSimB200_ShardGroup_RangeQueryBatchDevice on a 10M x 768 shard against VecSimB200_LabelRangeQueryBatchDevice alone.
In (b) and (c) 8 queries of the collective are checked against the unsharded answer: at one GPU the local call on the whole
corpus; on N GPUs every rank's local rows for them, gathered and merged on the host by the documented rule.

Run:  python bench_sharded_lists.py [--rows 10000000] [--steps 20]      (one GPU: the group of one is the local call)
      torchrun --nproc-per-node N bench_sharded_lists.py --gpus N        (N ranks, one exchange per step)
Prints one JSON line with the card's name, power limit and max SM clock beside the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers still stand; say what is missing
        return {"gpu": f"unknown ({e})"}


def timed(torch, fn, reps, stream):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    stream.synchronize()
    start.record(stream)
    for _ in range(reps):
        fn()
    stop.record(stream)
    stop.synchronize()
    return start.elapsed_time(stop) / reps


def merge_alone(env):
    """(a): synthetic sorted runs"""
    torch, L = env.torch, env.L
    out = []
    for G in (2, 4, 8):
        for w, range_query in ((10, 0), (1000, 0), (1024, 1), (4096, 1)):
            nq = 256
            n = nq * w
            block = int(L.VecSimB200_ShardListBlockBytes(nq, w))
            # top-w: full runs; range: runs adding up to exactly w, the largest union a range row can have
            m = [w] * G if not range_query else [w - (G - 1) * (w // G)] + [w // G] * (G - 1)
            g = torch.Generator(device=env.dev).manual_seed(G * 10 + w)
            blocks = torch.zeros((G, block), dtype=torch.uint8, device=env.dev)
            for r in range(G):
                sc = torch.sort(torch.rand((nq, w), generator=g, device=env.dev), dim=1).values
                lab = torch.randint(0, 1 << 40, (nq, w), generator=g, device=env.dev)
                cnt = torch.full((nq,), m[r], dtype=torch.int32, device=env.dev)
                blocks[r, :n * 8] = lab.view(torch.uint8).reshape(-1)
                blocks[r, n * 8:n * 12] = sc.view(torch.uint8).reshape(-1)
                blocks[r, n * 12:n * 12 + nq * 4] = cnt.view(torch.uint8).reshape(-1)
            ol_ = torch.empty((nq, w), dtype=torch.int64, device=env.dev)
            os_ = torch.empty((nq, w), dtype=torch.float32, device=env.dev)
            oc = torch.empty(nq, dtype=torch.int32, device=env.dev)

            def call():
                assert L.VecSimB200_MergeShardListBlocks(blocks.data_ptr(), G, nq, w, range_query, 0, ol_.data_ptr(), os_.data_ptr(),
                                                         oc.data_ptr(), env.sp) == 0

            ms = timed(torch, call, 200, env.stream)
            bytes_ = nq * (sum(m) * 12 + G * 4) + nq * (w * 12 + 4)  # every run and count read once, the rows written
            out.append({"G": G, "nq": nq, "w": w, "kind": "range" if range_query else "top-w", "kernel_ms": round(ms, 4),
                        "bytes": bytes_, "hbm_floor_share": round(bytes_ / HBM_BYTES_PER_S / (ms * 1e-3), 4)})
    return out


def host_merge(parts, w, range_query):
    """the documented merge rule on the host: parts = [(labels [nq, w], scores, counts)] per rank"""
    nq = parts[0][0].shape[0]
    lab = np.full((nq, w), -1, np.int64)
    sc = np.full((nq, w), np.nan, np.float32)
    cnt = np.zeros(nq, np.int64)
    for q in range(nq):
        cs = [int(p[2][q]) for p in parts]
        total = sum(cs)
        if any(c == 0xFFFFFFFF for c in cs):
            cnt[q] = 0xFFFFFFFF
            continue
        cnt[q] = min(total, 0xFFFFFFFF) if range_query else min(total, w)
        if range_query and total > w:
            continue
        items = sorted((np.float32(p[1][q, i]) + np.float32(0), int(p[0][q, i])) for p in parts for i in range(min(int(p[2][q]), w)))
        for i, (s, l_) in enumerate(items[:w]):
            lab[q, i], sc[q, i] = l_, s
    return lab, sc, cnt


def check_against_unsharded(env, got, local_rows, w, range_query, pick):
    """got: the collective's (labels, scores, counts) for queries `pick`; local_rows: this rank's local call for them"""
    torch = env.torch
    if env.world == 1:
        exp = local_rows
    else:
        gathered = []
        for a in local_rows:
            t = torch.from_numpy(np.ascontiguousarray(a)).to(env.dev)
            bufs = [torch.empty_like(t) for _ in range(env.world)]
            env.dist.all_gather(bufs, t)
            gathered.append([b.cpu().numpy() for b in bufs])
        exp = host_merge(list(zip(*gathered)), w, range_query)
    gl, gs, gc = got
    el, es, ec = exp
    ok = (gl == el).all() and (gc.astype(np.int64) == np.asarray(ec).astype(np.int64)).all()
    live = gl >= 0
    ok = ok and (gs[live] == es[live]).all()
    return bool(ok)


def build_filters(env, lists, pairs, P):
    nq = len(pairs)
    arrays = [(C.c_void_p * 2)(lists[a], lists[b]) for a, b in pairs]
    pp = (C.c_void_p * nq)(*[C.cast(a, C.c_void_p) for a in arrays])
    return arrays, pp, (C.c_size_t * nq)(*([2] * nq))


def config5(env, args, index, lo, hi):
    """(b): the host path of run_config5 against the device pipeline into the collective"""
    import bench_postings as bp
    from redisearch_b200 import postings as ps
    from redisearch_b200._lib import load_library

    torch, L, vs, sp = env.torch, env.L, env.vs, env.sp
    P = ps.lib()
    total, DIM, k = args.rows, 768, 10
    S = load_library("libsynth_b200.so")
    S.Synth_DocFreq.restype = C.c_uint64
    S.Synth_DocFreq.argtypes = [C.c_uint64, C.c_uint64]
    S.Synth_Postings.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    chunks = (total + 1023) // 1024
    scratch = torch.empty(2 * chunks + 16, dtype=torch.int32, device=env.dev)
    d_total = torch.zeros(4, dtype=torch.int32, device=env.dev)
    h_count = np.zeros(4, dtype=np.uint32)
    lists, keep = {}, []
    for r in sorted({r for pr in bp.HYBRID_TERM_PAIRS for r in pr}):
        cap = int(S.Synth_DocFreq(total, r) * 1.2) + 4096
        ids = torch.empty(cap, dtype=torch.int32, device=env.dev)
        fr = torch.empty(cap, dtype=torch.int32, device=env.dev)
        assert S.Synth_Postings(total, r, ids.data_ptr(), fr.data_ptr(), scratch.data_ptr(), d_total.data_ptr(), h_count.ctypes.data, sp) == 0
        n = int(h_count[0])
        a = int(torch.searchsorted(ids[:n], torch.tensor([lo], dtype=torch.int32, device=env.dev), right=True).item())
        b = int(torch.searchsorted(ids[:n], torch.tensor([hi], dtype=torch.int32, device=env.dev), right=True).item())
        sl_i, sl_f = ids[a:b].contiguous(), fr[a:b].contiguous()
        keep.append((sl_i, sl_f))
        lists[r] = P.II_PostingList_FromDevice(sl_i.data_ptr(), sl_f.data_ptr(), b - a)
        assert lists[r]
    g = env.shard_group()
    results = []
    for nq in (16, 256):
        pairs = [bp.HYBRID_TERM_PAIRS[i % len(bp.HYBRID_TERM_PAIRS)] for i in range(nq)]
        qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
        assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, 43, 0, nq, DIM, sp) == 0
        assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0
        torch.cuda.synchronize()
        qh = qdev.cpu().numpy().copy()
        arrays, lists_pp, n_lists = build_filters(env, lists, pairs, P)
        # today's host path
        block = int(L.VecSimB200_ShardBlockBytes(nq, k))
        h_block = torch.empty(block, dtype=torch.uint8, pin_memory=True)
        d_block = torch.empty(block, dtype=torch.uint8, device=env.dev)
        d_all = torch.empty(block * env.world, dtype=torch.uint8, device=env.dev)
        m_scores = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
        m_labels = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
        rs_out = (C.c_void_p * nq)()
        q_ptrs = (C.c_void_p * nq)(*[qh[i].ctypes.data for i in range(nq)])
        id_ptrs, id_counts, b_counts = (C.c_void_p * nq)(), (C.c_size_t * nq)(), (C.c_size_t * nq)()
        b_labels, b_scores = np.zeros((nq, k), dtype=np.uint64), np.zeros((nq, k), dtype=np.float64)

        def host_step():
            hb = h_block.numpy()
            lab = hb[: nq * k * 8].view(np.int64).reshape(nq, k)
            sc = hb[nq * k * 8: nq * k * 12].view(np.float32).reshape(nq, k)
            lab[:] = -1
            sc[:] = np.nan
            P.II_IntersectBatch(nq, lists_pp, n_lists, rs_out)
            for i in range(nq):
                m = P.II_ResultSet_Len(rs_out[i]) if rs_out[i] else 0
                id_counts[i] = m
                id_ptrs[i] = P.II_ResultSet_DeviceDocIds(rs_out[i]) if m else None
            assert L.VecSimB200_TopKFilteredBatch(index.h, q_ptrs, nq, k, id_ptrs, id_counts, b_labels.ctypes.data, b_scores.ctypes.data,
                                                  b_counts) == 0
            for i in range(nq):
                c_ = b_counts[i]
                lab[i, :c_] = b_labels[i, :c_].astype(np.int64)
                sc[i, :c_] = b_scores[i, :c_].astype(np.float32)
                if rs_out[i]:
                    P.II_ResultSet_Free(rs_out[i])
            if env.world == 1:
                return lab.copy()
            d_block.copy_(h_block, non_blocking=True)
            env.dist.all_gather_into_tensor(d_all, d_block)
            assert L.VecSimB200_MergeShardBlocks(d_all.data_ptr(), env.world, nq, k, m_scores.data_ptr(), m_labels.data_ptr(), sp) == 0
            return m_labels.cpu().numpy()

        # the device pipeline into the collective
        o_l = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
        o_s = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
        o_c = torch.empty(nq, dtype=torch.int32, device=env.dev)
        modes = np.zeros(nq, dtype=np.int32)
        sets = (C.c_void_p * nq)()

        def device_step():
            P.II_IntersectBatchDevice(nq, lists_pp, n_lists, sp, sets)
            ids = (C.c_void_p * nq)(*[P.II_ResultSet_DeviceDocIds(sets[i]) if sets[i] else None for i in range(nq)])
            cnts = (C.c_void_p * nq)(*[P.II_ResultSet_DeviceLen(sets[i]) if sets[i] else None for i in range(nq)])
            caps = (C.c_size_t * nq)(*[P.II_ResultSet_Capacity(sets[i]) if sets[i] else 0 for i in range(nq)])
            rc = L.VecSimB200_ShardGroup_HybridTopKBatchDevice(g, index.h, qdev.data_ptr(), nq, k, ids, cnts, caps, None, o_l.data_ptr(),
                                                               o_s.data_ptr(), o_c.data_ptr(), modes.ctypes.data, sp)
            assert rc == 0, rc
            for i in range(nq):
                if sets[i]:
                    P.II_ResultSet_FreeAfter(sets[i], sp)

        row = {"nq": nq}
        for name, fn in (("host_path", host_step), ("device_collective", device_step)):
            for _ in range(max(3, args.warmup)):
                fn()
            env.barrier()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
            row[name + "_ms"] = round(env.max_over_ranks((time.perf_counter() - t0) / args.steps) * 1e3, 3)
        # check: 8 queries of the collective against the unsharded answer
        device_step()
        torch.cuda.synchronize()
        pick = list(range(8))
        got = (o_l.cpu().numpy()[pick], o_s.cpu().numpy()[pick], o_c.cpu().numpy().view(np.uint32)[pick])
        P.II_IntersectBatchDevice(nq, lists_pp, n_lists, sp, sets)
        ids = (C.c_void_p * nq)(*[P.II_ResultSet_DeviceDocIds(sets[i]) if sets[i] else None for i in range(nq)])
        cnts = (C.c_void_p * nq)(*[P.II_ResultSet_DeviceLen(sets[i]) if sets[i] else None for i in range(nq)])
        caps = (C.c_size_t * nq)(*[P.II_ResultSet_Capacity(sets[i]) if sets[i] else 0 for i in range(nq)])
        lab, sc, cnt, md, rc = index.hybrid_topk_batch_device(qdev, k, list(ids), list(caps), counts=list(cnts), stream=env.stream)
        assert rc == 0
        torch.cuda.synchronize()
        for i in range(nq):
            if sets[i]:
                P.II_ResultSet_FreeAfter(sets[i], sp)
        local = (lab.cpu().numpy()[pick], sc.cpu().numpy()[pick], cnt.cpu().numpy().view(np.uint32)[pick])
        row["checked_queries"] = len(pick)
        row["equal_unsharded"] = check_against_unsharded(env, got, local, k, False, pick)
        row["host_labels_equal"] = bool((host_step()[pick] == got[0]).all())
        results.append(row)
    return results


def range_collective(env, args, index):
    """(c): 256 queries, radius at each query's 10th / 1000th neighbour, cap 4096"""
    torch, L, sp = env.torch, env.L, env.sp
    nq, DIM, cap = 256, 768, 4096
    qdev = torch.empty((nq, DIM), dtype=torch.float32, device=env.dev)
    assert env.S.Synth_FillRows(qdev.data_ptr(), DIM * 4, 0, 44, 0, nq, DIM, sp) == 0
    assert env.S.Synth_NormalizeRowsF32(qdev.data_ptr(), DIM * 4, nq, DIM, sp) == 0
    lab0 = torch.empty((nq, 1000), dtype=torch.int64, device=env.dev)
    sc0 = torch.empty((nq, 1000), dtype=torch.float32, device=env.dev)
    assert L.VecSimB200_TopKQueryBatchDevice(index.h, qdev.data_ptr(), nq, 1000, lab0.data_ptr(), sc0.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    kth = sc0.cpu().numpy()
    radii = np.array([kth[i, 9 if i % 2 else 999] for i in range(nq)], dtype=np.float32)
    if env.world > 1:  # one radius for every rank: rank 0's
        t = torch.from_numpy(radii).to(env.dev)
        env.dist.broadcast(t, 0)
        radii = t.cpu().numpy()
    rd = torch.from_numpy(radii).to(env.dev)
    g = env.shard_group()
    o_l = torch.empty((nq, cap), dtype=torch.int64, device=env.dev)
    o_s = torch.empty((nq, cap), dtype=torch.float32, device=env.dev)
    o_c = torch.empty(nq, dtype=torch.int32, device=env.dev)
    l_l, l_s, l_c = torch.empty_like(o_l), torch.empty_like(o_s), torch.empty_like(o_c)

    def local():
        assert L.VecSimB200_LabelRangeQueryBatchDevice(index.h, qdev.data_ptr(), nq, rd.data_ptr(), cap, 0, l_l.data_ptr(), l_s.data_ptr(),
                                                       l_c.data_ptr(), sp) == 0

    def collective():
        assert L.VecSimB200_ShardGroup_RangeQueryBatchDevice(g, index.h, qdev.data_ptr(), nq, rd.data_ptr(), cap, 0, o_l.data_ptr(),
                                                             o_s.data_ptr(), o_c.data_ptr(), sp) == 0

    row = {"nq": nq, "cap": cap}
    for name, fn in (("local_ms", local), ("collective_ms", collective)):
        for _ in range(max(3, args.warmup)):
            fn()
        env.barrier()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        row[name] = round(env.max_over_ranks((time.perf_counter() - t0) / args.steps) * 1e3, 3)
    local()
    collective()
    torch.cuda.synchronize()
    pick = list(range(8))
    got = (o_l.cpu().numpy()[pick], o_s.cpu().numpy()[pick], o_c.cpu().numpy().view(np.uint32)[pick])
    mine = (l_l.cpu().numpy()[pick], l_s.cpu().numpy()[pick], l_c.cpu().numpy().view(np.uint32)[pick])
    row["checked_queries"] = len(pick)
    row["equal_unsharded"] = check_against_unsharded(env, got, mine, cap, True, pick)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--rows", type=int, default=10_000_000, help="corpus rows of (b), and rows per shard of (c)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only-merge", action="store_true")
    args = ap.parse_args()
    from bench import Env, build_shard

    env = Env()
    assert env.world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE {env.world}"
    env.L.VecSimB200_SetCoarseMode(1)
    res = {"bench": "sharded_lists", "gpus": env.world, **card(), "merge": merge_alone(env)}
    if not args.only_merge:
        vs = env.vs
        lo, hi = (args.rows * env.rank) // env.world, (args.rows * (env.rank + 1)) // env.world
        index, _ = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, hi - lo, lo, dim=768)
        res["config5"] = config5(env, args, index, lo, hi)
        index.close()
        shard, _ = build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, args.rows, env.rank * args.rows, dim=768)
        res["range"] = range_collective(env, args, shard)
        shard.close()
    if env.rank == 0:
        print(json.dumps(res))
    env.close()


if __name__ == "__main__":
    main()
