"""Multi-start solves on a crowded configs[2]-style world: how the fraction of solved problems grows with the seeds per
problem G, and what stopping the siblings of a converged seed (group_stop) saves.

The world is configs[2] with more and larger obstacles (40 spheres of radius 0.12 m instead of 8 of 0.10 m), so that a
single straight-line seed often ends infeasible.  Each of P problems is solved with G seeds (problems.with_seeds: seed 0
the straight line, the others through a random mid waypoint), with group_stop off and on.  Per setting: the fraction of
problems with a converged seed, the device time of a batch (CUDA events around tb200_solve_batch's launches), solved
problems per second, and the seeds that were stopped by their group.  The card, its power limit and SM clocks are read
in the same run.

    python scripts/multi_start.py [--problems 128] [--seeds 1,4,8] [--reps 3] [--out results/multi_start.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, problems, sharding  # noqa: E402


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
    ap.add_argument("--problems", type=int, default=128)
    ap.add_argument("--seeds", default="1,4,8")
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--obstacles", type=int, default=40)
    ap.add_argument("--radius", type=float, default=0.12)
    ap.add_argument("--spread", type=float, default=0.6, help="rad: half width of the mid-waypoint box of seeds > 0")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    base = problems.config2(B=a.problems, T=a.T, n_obstacles=a.obstacles, obstacle_radius=a.radius)
    rows = []
    for G in (int(s) for s in a.seeds.split(",")):
        d = problems.with_seeds(base, G, np.random.default_rng(20261016), a.spread)
        for stop in ((0, 1) if G > 1 else (0,)):
            p = api.Problem(d)
            p.set_groups(G, stop)
            p.solve()  # warm-up: module load, first launches
            ms, solved, stopped, status = [], [], [], None
            for _ in range(a.reps):
                r = p.solve()
                g = p.group_results()
                if status is not None and not stop:  # deterministic; with group_stop the stopped seeds are not
                    assert (r["status"] == status).all()
                status = r["status"]
                ms.append(r["timing"]["total_ms"])
                solved.append(sharding.converged_count(r["status"], G))
                stopped.append(int((g["ended_by"] == 2).sum()))
            p.close()
            med = float(np.median(ms))
            row = dict(G=G, group_stop=stop, problems=a.problems, trajectories=d.B, solved=solved[0],
                       solved_fraction=solved[0] / a.problems, device_ms=med, device_ms_all=ms,
                       solved_per_s=solved[0] / (med * 1e-3), seeds_stopped_by_group=stopped[0])
            rows.append(row)
            print(json.dumps(row), flush=True)
    info = gpu_info()
    print(json.dumps({"gpu": info}))
    print(f"\n{'G':>2} {'stop':>4} {'solved':>8} {'device ms':>10} {'solved/s':>9} {'stopped':>8}")
    for r in rows:
        print(f"{r['G']:>2} {r['group_stop']:>4} {r['solved_fraction']:>8.3f} {r['device_ms']:>10.1f} "
              f"{r['solved_per_s']:>9.1f} {r['seeds_stopped_by_group']:>8}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "args": vars(a), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
