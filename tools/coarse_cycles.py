#!/usr/bin/env python
"""Cycle account of the fixed-bound main pass of the batched fp32 KNN scan (coarse_wgmma_kernel<false,*,*,1>, over the int8
copy at the flagship shape).

Builds libvecsim_b200.so with -DCOARSE_CYCLE_ACCOUNT into a directory of its own (never redisearch_b200/lib/), runs the
flagship shape of bench.py (FLAT 10M x 768 fp32 cosine, k=10, batch 256; bench.py's generators and seeds) and prints,
per counter, the median and p90 over CTAs as a share of the pass, next to the median cycles per tile.  The counters are
clock64() sums kept per CTA and role (consumer warpgroup 0 / 1, producer warp); the default build compiles none of it.

    python tools/coarse_cycles.py [--lib-dir DIR] [--rows N] [--batch B] [--out FILE]

--lib-dir: use an instrumented library already built there (make -C redisearch_b200/csrc OUT=DIR OBJ=DIR/obj
EXTRA_NVFLAGS=-DCOARSE_CYCLE_ACCOUNT DIR/libvecsim_b200.so); without it the library is built in a temporary directory.
Needs a GPU.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = ["pass", "wait", "issue", "wait1", "epilogue", "handoff", "tiles"]  # kCa* in coarse_tc.cu
MAX_CTAS = 1024
ROLES = 3  # consumer warpgroup 0, consumer warpgroup 1, producer


def build(out_dir):
    obj = os.path.join(out_dir, "obj")
    os.makedirs(obj, exist_ok=True)
    target = os.path.join(out_dir, "libvecsim_b200.so")
    subprocess.run(["make", "-j", str(min(8, os.cpu_count() or 1)), target, f"OUT={out_dir}", f"OBJ={obj}",
                    "EXTRA_NVFLAGS=-DCOARSE_CYCLE_ACCOUNT"], cwd=os.path.join(ROOT, "redisearch_b200", "csrc"), check=True,
                   stdout=subprocess.DEVNULL)
    return target


def quantile(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * (len(xs) - 1) + 0.5))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-dir", default=None)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default=None, help="also write the table as JSON here")
    args = ap.parse_args()

    tmp = None
    if args.lib_dir:
        path = os.path.join(args.lib_dir, "libvecsim_b200.so")
    else:
        tmp = tempfile.mkdtemp(prefix="coarse_cycles_")
        path = build(tmp)
    from redisearch_b200 import _lib

    _lib._cache["libvecsim_b200.so"] = C.CDLL(path)  # the instrumented library in place of the in-tree one
    import bench

    env = bench.Env()
    torch, L, vs, S, sp = env.torch, env.L, env.vs, env.S, env.sp
    L.VecSimB200_CoarseCycles.argtypes = [C.c_void_p, C.c_int]
    L.VecSimB200_CoarseCycles.restype = C.c_int
    index, _ = bench.build_shard(env, vs.VecSimType_FLOAT32, vs.VecSimMetric_Cosine, args.rows, 0)
    nq, dim, k = args.batch, bench.DIM, bench.K
    q = torch.empty((nq, dim), dtype=torch.float32, device=env.dev)
    assert S.Synth_FillRows(q.data_ptr(), dim * 4, 0, bench.SEED_QUERIES, 0, nq, dim, sp) == 0
    assert S.Synth_NormalizeRowsF32(q.data_ptr(), dim * 4, nq, dim, sp) == 0
    labels = torch.empty((nq, k), dtype=torch.int64, device=env.dev)
    scores = torch.empty((nq, k), dtype=torch.float32, device=env.dev)
    for _ in range(3):  # the counters hold the last main pass
        assert L.VecSimB200_TopKQueryBatchDevice(index.h, q.data_ptr(), nq, k, labels.data_ptr(), scores.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    host = (C.c_ulonglong * (MAX_CTAS * ROLES * len(SLOTS)))()
    assert L.VecSimB200_CoarseCycles(host, MAX_CTAS) == len(SLOTS)
    v = [host[i] for i in range(len(host))]

    def at(cta, role, slot):
        return v[(cta * ROLES + role) * len(SLOTS) + SLOTS.index(slot)]

    ctas = [c for c in range(MAX_CTAS) if at(c, 2, "pass") > 0]
    table = {"gpu": torch.cuda.get_device_name(0), "ctas": len(ctas), "rows": args.rows, "batch": nq, "roles": {}}
    for role, name in [(0, "consumer warpgroup 0"), (1, "consumer warpgroup 1"), (2, "producer")]:
        live = [c for c in ctas if at(c, role, "pass") > 0]
        if not live:
            continue
        # the producer fills the ring once for every tile of the CTA; a consumer warpgroup counts the tiles it multiplies
        tiles = [at(c, role, "tiles") for c in live]
        rows = {}
        for slot in SLOTS[:-1]:
            share = [at(c, role, slot) / at(c, role, "pass") for c in live]
            per_tile = [at(c, role, slot) / max(1, t) for c, t in zip(live, tiles)]
            rows[slot] = {"share_median": quantile(share, 0.5), "share_p90": quantile(share, 0.9),
                          "clk_per_tile_median": quantile(per_tile, 0.5)}
        table["roles"][name] = {"ctas": len(live), "tiles_median": quantile(tiles, 0.5), "counters": rows}
        print(f"{name}: {len(live)} CTAs, median {quantile(tiles, 0.5)} tiles per {'CTA' if role == 2 else 'warpgroup'}")
        print(f"  {'counter':10s} {'median':>8s} {'p90':>8s} {'clk/tile':>10s}")
        for slot, r in rows.items():
            print(f"  {slot:10s} {r['share_median']:8.3f} {r['share_p90']:8.3f} {r['clk_per_tile_median']:10.0f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(table, f, indent=1)
    if tmp:
        subprocess.run(["rm", "-rf", tmp], check=False)


if __name__ == "__main__":
    main()
