#!/usr/bin/env python
"""Time per kernel in one step of the flagship workload (bench.py's default config: FLAT 10M x 768 fp32 cosine, k=10,
batch 256, one GPU), from torch.profiler with CUDA activities, in a run of its own.

Builds the index and the queries as bench.py does (its generators and seeds), warms up, then profiles --steps device
steps (VecSimB200_ShardGroup_TopKBatchDevice, as bench.py times them) and prints, per kernel name, the launches and the
device time per step, largest first, with the sum over all kernels and the wall time per step under the profiler.

    python tools/step_kernels.py [--rows N] [--batch B] [--steps S] [--out FILE]

--out also writes the table as JSON.  Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the table as JSON here")
    args = ap.parse_args()

    import bench
    from torch.profiler import ProfilerActivity, profile

    env = bench.Env()
    torch, L, vs, S, sp = env.torch, env.L, env.vs, env.S, env.sp
    index, _ = bench.build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, args.rows, 0)
    group = env.shard_group()
    nq, dim, k = args.batch, bench.DIM, bench.K
    q = torch.empty((nq, dim), dtype=torch.float32, device=env.dev)
    assert S.Synth_FillRows(q.data_ptr(), dim * 4, 0, bench.SEED_QUERIES, 0, nq, dim, sp) == 0
    assert S.Synth_NormalizeRowsF32(q.data_ptr(), dim * 4, nq, dim, sp) == 0
    labels = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
    scores = torch.empty((nq, k), dtype=torch.float32, device=env.dev)

    def step():
        assert L.VecSimB200_ShardGroup_TopKBatchDevice(group, index.h, q.data_ptr(), nq, k, labels.data_ptr(), scores.data_ptr(), sp) == 0

    for _ in range(max(1, args.warmup)):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1000.0 / args.steps

    per = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        name = e.name
        c = per.setdefault(name, {"launches": 0, "us": 0.0})
        c["launches"] += 1
        c["us"] += us
    rows = sorted(per.items(), key=lambda kv: -kv[1]["us"])
    total_us = sum(v["us"] for _, v in rows) / args.steps
    table = {"gpu": torch.cuda.get_device_name(0), "rows": args.rows, "batch": nq, "k": k, "steps": args.steps,
             "wall_ms_per_step_under_profiler": wall_ms, "kernel_us_per_step": total_us, "kernels": []}
    print(f"{table['gpu']}: {args.rows} x {dim}, batch {nq}, k {k}, {args.steps} steps")
    print(f"  {'us/step':>10s} {'share':>6s} {'launches/step':>14s}  kernel")
    for name, v in rows:
        us = v["us"] / args.steps
        table["kernels"].append({"name": name, "us_per_step": us, "launches_per_step": v["launches"] / args.steps})
        print(f"  {us:10.1f} {us / total_us:6.3f} {v['launches'] / args.steps:14.1f}  {name[:140]}")
    print(f"  {total_us:10.1f} {'':6s} {'':14s}  all kernels; wall {wall_ms * 1000.0:.1f} us per step under the profiler")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(table, f, indent=1)


if __name__ == "__main__":
    main()
