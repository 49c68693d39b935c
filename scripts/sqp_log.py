"""What the SQP iteration log costs (DESIGN.md sections 4.7 and 7): configs[2], batch 1024, three cases - log off, log
without the points, log with the points - each the median of three solves on one handle after a warm-up solve.

Per case: device time of the solve (CUDA events around tb200_solve_batch's launches), records per trajectory, the bytes
the records take on the device, and whether every result array is bit-identical to the log-off solve.  The card, its
power limit and SM clocks are read in the same run.

    python scripts/sqp_log.py [--B 1024] [--T 30] [--capacity 256] [--reps 3] [--out results/sqp_log.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, problems  # noqa: E402

KEYS = ("x", "status", "total_cost", "cost_vals", "cnt_viols", "n_qp_solves", "n_func_evals", "n_admm_iters")


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
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--capacity", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    d = problems.config2(B=a.B, T=a.T)
    p = api.Problem(d)
    L = p.layout
    rows, ref = [], None
    try:
        for name, cap, with_x in (("off", 0, False), ("log", a.capacity, False), ("log+x", a.capacity, True)):
            p.set_sqp_log(cap, with_x)
            p.solve()  # warm-up: module load, first launches, the log buffer
            ms, same = [], True
            for _ in range(a.reps):
                r = p.solve()
                ms.append(r["timing"]["total_ms"])
                if ref is None:
                    ref = r
                same &= all(r[k].tobytes() == ref[k].tobytes() for k in KEYS)
            row = dict(case=name, device_ms=float(np.median(ms)), ms=ms, identical=bool(same))
            if cap:
                log = p.sqp_log()
                stride = 16 + 3 * L.n_cnts + 2 * L.n_costs + (d.T * d.D if with_x else 0)
                n = log["n_records"]
                row.update(records_per_traj=float(n.mean()), records_max=int(n.max()), dropped=int(log["n_dropped"].sum()),
                           bytes_per_record=8 * stride, bytes_written=int(8 * stride * n.sum()))
            rows.append(row)
            print(json.dumps(row))
    finally:
        p.close()
    off = rows[0]["device_ms"]
    for row in rows[1:]:
        row["overhead_pct"] = 100.0 * (row["device_ms"] - off) / off
    out = dict(config=f"configs[2] B={a.B} T={a.T}", capacity=a.capacity, reps=a.reps, gpu=gpu_info(), rows=rows)
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
