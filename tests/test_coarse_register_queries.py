"""GPU: the fixed-bound main pass with the leading K blocks of its queries held in registers (coarse_tc.cu kRegKb).

Where the plan holds register blocks (cosine / inner product, dims whose K-block count frees a ring stage, e.g. 520 -> 9 blocks
padded to 10, 768, 1024), every approximate distance must be the same fp16 x fp16 -> fp32 wgmma sequence as with all blocks in
shared memory.  So for each batch, run in a subprocess because VECSIM_B200_REGKB is read once per process:
  - labels and score bits equal the exact scan's (VecSimB200_SetCoarseMode(0));
  - the per-query tiers (VecSimB200_LastCoarseFlags) are identical with VECSIM_B200_REGKB=0 and with the default.
Squared L2 and filtered batches hold no register blocks; L2 is checked here that it still plans and answers as before.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# metric, rows, dim, batch, k; batch sizes leave empty query slots in the last group of 64 (17, 200) or none (256)
CASES = [
    ("cosine", 66_000, 520, 17, 10),
    ("cosine", 66_000, 768, 256, 10),
    ("cosine", 66_000, 1024, 200, 10),
    ("cosine", 70_000, 384, 200, 16),
    ("ip", 66_000, 768, 200, 10),
    ("ip", 66_000, 520, 256, 10),
    ("l2", 66_000, 768, 17, 10),
]

_SCRIPT = r"""
import ctypes as C, sys, os
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch, oracle_lib as ol
from redisearch_b200 import vecsim as vs

metrics = {"cosine": vs.VecSimMetric_Cosine, "ip": vs.VecSimMetric_IP, "l2": vs.VecSimMetric_L2}

def batch(g, qd, nq, k):
    out_l = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert vs.lib().VecSimB200_TopKQueryBatchDevice(g.h, qd.data_ptr(), nq, k, out_l.data_ptr(), out_s.data_ptr(), sp) == 0
    torch.cuda.synchronize()
    flags = np.zeros(nq, dtype=np.uint32)
    frc = vs.lib().VecSimB200_LastCoarseFlags(g.h, flags.ctypes.data, nq)
    return out_l.cpu().numpy(), out_s.cpu().numpy(), flags, frc

res = {}
for ci, (metric, n, dim, nq, k) in enumerate(CASES):
    rows = ol.synth_rows(ol.F32, 42, 0, n, dim)
    g = vs.VecSimIndex(vs.VecSimType_FLOAT32, dim, metrics[metric])
    assert g.add_many(rows, label0=1) == n
    qs = ol.synth_rows(ol.F32, 43, 0, nq, dim)
    if metric == "cosine":
        for i in range(nq):
            ol.port().orc_normalize(ol._p(qs[i]), dim, ol.F32)
    qd = torch.from_numpy(np.ascontiguousarray(qs)).cuda()
    vs.lib().VecSimB200_SetCoarseMode(1)
    l, s, f, frc = batch(g, qd, nq, k)
    vs.lib().VecSimB200_SetCoarseMode(0)
    el, es, _, _ = batch(g, qd, nq, k)
    vs.lib().VecSimB200_SetCoarseMode(-1)
    res[f"l{ci}"], res[f"s{ci}"], res[f"f{ci}"], res[f"frc{ci}"] = l, s, f, np.int64(frc)
    res[f"el{ci}"], res[f"es{ci}"] = el, es
    del g
np.savez(OUT, **res)
print("REGKB-OK")
"""


def _run(tmp_path, cap):
    out = str(tmp_path / f"regkb_{cap or 'default'}.npz")
    code = f"ROOT = {ROOT!r}\nOUT = {out!r}\nCASES = {CASES!r}\n" + _SCRIPT
    env = dict(os.environ)
    env.pop("VECSIM_B200_REGKB", None)
    if cap is not None:
        env["VECSIM_B200_REGKB"] = cap
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1200, env=env)
    assert r.returncode == 0 and "REGKB-OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    return np.load(out)


def test_register_held_queries_keep_every_distance(tmp_path):
    regs, smem = _run(tmp_path, None), _run(tmp_path, "0")
    for ci, (metric, n, dim, nq, k) in enumerate(CASES):
        case = (metric, n, dim, nq, k)
        for r in (regs, smem):
            assert int(r[f"frc{ci}"]) == 0, f"{case}: the batch did not take the tensor-core path"
            assert (r[f"f{ci}"] != 0).sum() >= nq * 0.9, f"{case}: tiers {np.bincount(r[f'f{ci}'], minlength=3).tolist()}"
            # the exact scan's answer, bit for bit
            assert (r[f"l{ci}"] == r[f"el{ci}"]).all(), case
            assert r[f"s{ci}"].tobytes() == r[f"es{ci}"].tobytes(), case
        # the same approximate distances: every query proven on the same tier
        assert (regs[f"f{ci}"] == smem[f"f{ci}"]).all(), (case, regs[f"f{ci}"], smem[f"f{ci}"])
        assert (regs[f"l{ci}"] == smem[f"l{ci}"]).all() and regs[f"s{ci}"].tobytes() == smem[f"s{ci}"].tobytes(), case
