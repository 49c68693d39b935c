"""Schedule of one solve by the persistent SQP kernel: when trajectories finish, how busy the SMs were, and whether
the last trajectory ran uninterrupted (then the batch is bound by that trajectory's own length)."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from trajopt_b200 import api, problems
cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
d = {"cfg1": problems.config1, "cfg2": problems.config2, "cfg3": problems.config3}[cfg](B=B, T=30)
p = api.Problem(d)
for rep in range(2):
    got = p.solve()
tm = got["timing"]
buf = np.zeros(1 + 2 * B, np.uint64)
p.lib.tb200_debug_schedule(p.handle, buf.ctypes.data_as(C.POINTER(C.c_uint64)))
t0 = float(buf[0]); fin = (buf[1:1 + B].astype(np.float64) - t0) * 1e-6; busy = buf[1 + B:].astype(np.float64) * 1e-6
it = got["n_admm_iters"].astype(np.float64)
print(f"{cfg} B={B}: total {tm['total_ms']:.1f} ms; converged {(got['status'] == 0).sum()}; ADMM iterations {it.sum():.0f} (max {it.max():.0f})")
print("finish time percentiles (ms): " + " ".join(f"p{q}={np.percentile(fin, q):.0f}" for q in (10, 50, 90, 99, 100)))
import torch
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
print(f"SM busy time {busy.sum():.0f} ms = {busy.sum() / (n_sm * fin.max()) * 100:.0f}% of {n_sm} SMs x {fin.max():.0f} ms; ns per ADMM iteration (busy / iterations): {busy.sum() * 1e6 / it.sum():.0f}")
last = np.argsort(-fin)[:8]
for b in last:
    print(f"  traj {b}: finished {fin[b]:.0f} ms, busy {busy[b]:.0f} ms ({100 * busy[b] / fin[b]:.0f}% of its life), {it[b]:.0f} iterations, {got['n_qp_solves'][b]} QPs, status {got['status'][b]}")
longest = np.argsort(-busy)[:5]
print("longest by busy time:", [(int(b), round(float(busy[b])), round(float(fin[b]))) for b in longest])
