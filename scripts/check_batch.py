"""Collision check of a solved configs[2] batch (tb200_check_trajectories): how long the check takes, and how many
OPT_CONVERGED trajectories are in contact between their waypoints.

configs[2] carries a DISCRETE collision constraint: its rows exist only at the waypoints, so a converged trajectory can
still sweep through an obstacle between two of them.  The script solves the batch, then checks the solution (x = None: the
solve's x, already on the device) with each type at margin 0 (LVS types at --lvs) and reports per type:
  * the kernel time of one check, from torch.profiler's CUDA activity (the slot kernel plus the per-trajectory summary),
    in a profiled run of its own;
  * the wall time of one tb200_check_trajectories call (host clock around calls that end in a stream synchronise),
    median over --reps calls with the profiler off;
  * the trajectories in contact, and how many of them ended OPT_CONVERGED.
The card, its power limit and SM clocks are read in the same run.

    python scripts/check_batch.py [--batch 1024] [--lvs 0.01] [--reps 20] [--out results/check_batch.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, capi, problems  # noqa: E402

TYPES = {"DISCRETE": capi.COLL_DISCRETE, "LVS_DISCRETE": capi.COLL_LVS_DISCRETE, "CONTINUOUS": capi.COLL_CONTINUOUS,
         "LVS_CONTINUOUS": capi.COLL_LVS_CONTINUOUS}
KERNELS = ("check_trajectories_kernel", "check_summary_kernel")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return {"nvidia_smi": "unavailable"}
    return dict(zip(q.split(","), (v.strip() for v in out.split(","))))


def kernel_us_per_call(p, type, lvs, reps):
    """Device time of the check's kernels per call (µs), from torch.profiler's CUDA activity over `reps` calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            p.check(None, type=type, lvs=lvs)
        torch.cuda.synchronize()
    total, launches = 0.0, 0
    for e in prof.events():
        if any(k in e.name for k in KERNELS):
            total += e.device_time_total
            launches += 1
    if launches == 0:
        raise RuntimeError("torch.profiler recorded no check kernel: the kernel time is not measured")
    return total / reps, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--lvs", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    d = problems.config2(B=a.batch, T=a.T)
    p = api.Problem(d)
    p.solve_resident()
    res = p.fetch()
    converged = res["status"] == capi.OPT_CONVERGED
    rows = []
    for name, type in TYPES.items():
        r = p.check(None, type=type, lvs=a.lvs)  # warm-up (module load, first launch) and the answer
        ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            p.check(None, type=type, lvs=a.lvs)
            ms.append((time.perf_counter() - t0) * 1e3)
        rows.append(dict(type=name, lvs=a.lvs if "LVS" in name else None, margin=0.0, call_ms=float(np.median(ms)),
                         call_ms_all=ms, in_contact=int(r["in_collision"].sum()),
                         converged=int(converged.sum()), converged_in_contact=int((r["in_collision"] & converged).sum()),
                         min_distance_of_converged=float(np.min(r["min_distance"][converged])) if converged.any() else None))
    for row in rows:  # profiled runs of their own
        row["kernel_us"], row["kernel_launches"] = kernel_us_per_call(p, TYPES[row["type"]], a.lvs, a.reps)
        print(json.dumps(row), flush=True)
    p.close()
    info = gpu_info()
    print(json.dumps({"gpu": info}))
    print(f"\nconfigs[2], batch {a.batch}, T {a.T}: {int(converged.sum())} trajectories OPT_CONVERGED")
    print(f"{'type':>15} {'kernel us':>10} {'call ms':>8} {'in contact':>11} {'converged in contact':>21}")
    for r in rows:
        print(f"{r['type']:>15} {r['kernel_us']:>10.1f} {r['call_ms']:>8.3f} {r['in_contact']:>11} {r['converged_in_contact']:>21}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "args": vars(a), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
