"""Throughput per joint count: the configs[2] term mix (tests/test_shape_sweep.build_case: JointVel + JointAcc costs, a
CartPose constraint at the last waypoint, discrete collision constraints against 8 obstacle spheres per trajectory) on
the robot of every joint count from 1 to 16 (trajopt_b200.robots.BY_JOINT_COUNT, and test_shape_sweep's robots of 3
and 6 joints), B trajectories of T waypoints, solved on one
GPU.  Per count it reports the device time of each solve (CUDA events around it, tb200_last_timing), the converged
count and converged trajectories per second.  The card and its power limit are read in the same run.

    python scripts/joint_counts.py [--batch 1024] [--T 30] [--reps 2] [--out results/joint_counts.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from unittest import mock  # noqa: E402

from trajopt_b200 import api, capi, robots  # noqa: E402
import test_shape_sweep  # noqa: E402  (build_case: the configs[2] term mix on a robot of its table)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return {"nvidia_smi": "unavailable"}
    return dict(zip(q.split(","), (v.strip() for v in out.split(","))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2, help="timed solves per count (after one warm-up solve)")
    ap.add_argument("--counts", default="1-16", help="joint counts, e.g. 1-16 or 4,8,16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if "-" in a.counts:
        lo, hi = (int(v) for v in a.counts.split("-"))
        counts = list(range(lo, hi + 1))
    else:
        counts = [int(v) for v in a.counts.split(",")]
    rows = []
    for D in counts:
        with mock.patch.dict(test_shape_sweep.ROBOTS, robots.BY_JOINT_COUNT):  # (3 and 6 joints: the sweep's own)
            d = test_shape_sweep.build_case(D, a.T, B=a.batch, seed=1000 + D)
        p = api.Problem(d)
        try:
            p.solve()  # warm-up
            ms, conv = [], []
            for _ in range(a.reps):
                r = p.solve()
                ms.append(r["timing"]["total_ms"])
                conv.append(int((r["status"] == capi.OPT_CONVERGED).sum()))
        finally:
            p.close()
        row = {"D": D, "device_ms": ms, "converged": conv,
               "converged_per_s": [c / (t * 1e-3) for c, t in zip(conv, ms)]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    report = {"gpu": gpu_info(), "config": "configs[2] term mix (build_case)", "batch": a.batch, "T": a.T, "counts": rows}
    print(json.dumps(report, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
