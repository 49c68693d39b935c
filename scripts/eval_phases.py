"""Cycles of thread 0 between the block barriers of the convexify kernel (needs a TB200_EVAL_PROFILE build)."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from trajopt_b200 import api, problems
B = 1024
d = problems.config2(B=B, T=30)
p = api.Problem(d)
x = d.init_traj + 0.05 * np.random.default_rng(0).standard_normal(d.init_traj.shape)
p.convexify_timed(x)
p.lib.tb200_debug_eval_prof(None, 1)
n = 4
for k in range(n):
    tm = p.convexify_timed(x)
prof = np.zeros(16, np.uint64)
p.lib.tb200_debug_eval_prof(prof.ctypes.data_as(C.POINTER(C.c_uint64)), 0)
names = {1: "load x / obstacles", 2: "FK local frames", 3: "FK chain products", 4: "emission (A/B, centres)", 5: "cart rows + collision rows",
         6: "joint terms", 7: "object values (in-order sums)"}
tot = prof.sum()
print(f"launch {tm['convexify_ms']*1e3:.1f} us; mean cycles per CTA {tot / (n * B):.0f}")
for k, nm in names.items():
    print(f"  {nm:34s} {prof[k] / (n * B):8.0f} cycles  {100.0 * prof[k] / tot:5.1f}%")
# ---- per-CTA timeline of the last launch
tr = np.zeros(3 * 4096, np.uint64)
p.lib.tb200_debug_eval_prof(tr.ctypes.data_as(C.POINTER(C.c_uint64)), 2)
tr = tr.reshape(4096, 3)[:B].astype(np.float64)
t0 = tr[:, 0].min()
st, en, smid = (tr[:, 0] - t0) * 1e-3, (tr[:, 1] - t0) * 1e-3, tr[:, 2].astype(int)
dur = en - st
print(f"timeline: first start 0, last end {en.max():.1f} us; CTA duration us: mean {dur.mean():.1f} p10 {np.percentile(dur,10):.1f} p50 {np.percentile(dur,50):.1f} p90 {np.percentile(dur,90):.1f} max {dur.max():.1f}")
print("CTA starts (us) percentiles:", " ".join(f"p{q}={np.percentile(st,q):.1f}" for q in (1, 25, 50, 58, 60, 75, 99)))
import torch
per_sm = np.bincount(smid, minlength=torch.cuda.get_device_properties(0).multi_processor_count)
print("CTAs per SM: min", per_sm.min(), "max", per_sm.max(), "SMs used", (per_sm > 0).sum())
grid = np.linspace(0, en.max(), 21)
print("resident CTAs over time:", " ".join(f"{((st <= g) & (en > g)).sum()}" for g in grid))
