"""The configs[4] trust-region sweep (problems.CONFIG4_SWEEP: 4 trust box sizes x 2 shrink ratios x 3 expand ratios = 24
points) solved two ways on one GPU:

  separate  one problem of B trajectories, solved 24 times, once per sweep point (tb200_problem_set_sqp_params);
  table     one problem of 24 * B trajectories (problems.sweep), every tile under its own point, solved once.

The script asserts that every trajectory's results (x, status, costs, violations, QP / function / ADMM counts) are
identical between the two: configs[4] uses discrete collision, so the layout does not depend on the batch.  Per way it
reports the device time (CUDA events around the solve, tb200_last_timing), the converged count per sweep point and
trajectories per second.  The card, its power limit and SM clocks are read in the same run.

    python scripts/param_sweep.py [--batch 256] [--T 40] [--reps 2] [--out results/param_sweep.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, capi, problems  # noqa: E402

RESULT_KEYS = ("x", "status", "total_cost", "cost_vals", "cnt_viols", "n_qp_solves", "n_func_evals", "n_admm_iters")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,memory.used"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return {"nvidia_smi": "unavailable"}
    return dict(zip(q.split(","), (v.strip() for v in out.split(","))))


def sweep_params():
    out = []
    for tb, sh, ex in problems.CONFIG4_SWEEP:
        p = capi.default_sqp_params()
        p.trust_box_size, p.trust_shrink_ratio, p.trust_expand_ratio = tb, sh, ex
        out.append(p)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="trajectories per sweep point")
    ap.add_argument("--T", type=int, default=40)
    ap.add_argument("--reps", type=int, default=2, help="timed repetitions of each way (the first solve warms up)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sets = sweep_params()
    K = len(sets)
    d = problems.config4(B=a.batch, T=a.T)
    tiled, idx = problems.sweep(d, sets)

    sep = api.Problem(d)
    tab = api.Problem(tiled)
    info_load = None

    def run_separate():
        res, ms = [], 0.0
        for p in sets:
            sep.set_sqp_params(p)
            r = sep.solve()
            ms += r["timing"]["total_ms"]
            res.append(r)
        return {k: np.concatenate([r[k] for r in res]) for k in RESULT_KEYS}, ms

    def run_table():
        nonlocal info_load
        r = tab.solve()
        info_load = gpu_info()  # (memory.used with both problems resident)
        return {k: r[k] for k in RESULT_KEYS}, r["timing"]["total_ms"]

    run_separate(), run_table()  # warm-up
    t_sep, t_tab = [], []
    for _ in range(a.reps):  # alternating
        s_res, ms = run_separate()
        t_sep.append(ms)
        t_res, ms = run_table()
        t_tab.append(ms)
    for k in RESULT_KEYS:
        assert s_res[k].tobytes() == t_res[k].tobytes(), f"{k} differs between the two ways"
    conv = [int((t_res["status"][idx == k] == capi.OPT_CONVERGED).sum()) for k in range(K)]
    n = K * a.batch
    report = {
        "gpu": gpu_info(), "gpu_after_table_solve": info_load, "config": "cfg4", "batch_per_point": a.batch, "T": a.T,
        "points": K, "trajectories": n, "identical": True,
        "separate": {"device_ms": t_sep, "traj_per_s": [n / (ms * 1e-3) for ms in t_sep]},
        "table": {"device_ms": t_tab, "traj_per_s": [n / (ms * 1e-3) for ms in t_tab]},
        "converged_per_point": [{"trust_box_size": tb, "trust_shrink_ratio": sh, "trust_expand_ratio": ex, "converged": c}
                                for (tb, sh, ex), c in zip(problems.CONFIG4_SWEEP, conv)],
    }
    print(json.dumps(report, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
