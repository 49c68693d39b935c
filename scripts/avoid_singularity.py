"""Device time of configs[2] with and without an avoid_singularity term on every waypoint (cost, then constraint), and
the evaluation step's share of it from the persistent kernel's timers (tb200_timing): DESIGN.md section 7.

    python scripts/avoid_singularity.py [--batch 1024] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, capi, problems  # noqa: E402


def variant(kind, B):
    d = problems.config2(B=B)
    if kind == "none":
        return d
    role = capi.ROLE_COST if kind == "cost" else capi.ROLE_CNT
    t = problems.avoid_singularity_term(role, 0, d.T - 1, d.robot_spec["tool"])
    return capi.ProblemDesc(d.robot_spec, d.T, list(d.terms) + [t], d.init_traj, fixed_timesteps=list(d._fixed_t),
                            fixed_dofs=list(d._fixed_d), cart_targets=d.cart_targets, obstacles=d.obstacles,
                            sqp=d.c.sqp, qp=d.c.qp)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    out = dict(card=card, batch=a.batch)
    for kind in ("none", "cost", "cnt"):
        d = variant(kind, a.batch)
        p = api.Problem(d)
        p.solve()  # warm-up
        rows = []
        for _ in range(a.repeats):
            r = p.solve()
            tm = r["timing"]
            rows.append(tm)
        p.close()
        keys = [k for k in rows[0] if isinstance(rows[0][k], (int, float))]
        out[kind] = {k: float(np.median([r[k] for r in rows])) for k in keys}
        out[kind]["converged"] = int((r["status"] == capi.OPT_CONVERGED).sum())
        out[kind]["qp_solves_mean"] = float(r["n_qp_solves"].mean())
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
