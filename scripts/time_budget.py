"""What a time limit (sqp max_time) buys on a batch: configs[2] at batch 1024 x 30 waypoints solved once without a
limit (device time T0, converged count), then with budgets of 0.1, 0.25, 0.5 and 0.75 x T0.  Per budget: converged and
OPT_TIME_LIMIT counts, device time, and the largest overshoot of a trajectory's finish time past the deadline (the QP
and evaluation already running when the limit passes are not interrupted).  Times come from %globaltimer (clock start
and finish times of the last solve) and CUDA events (device time).

    python scripts/time_budget.py [--B 1024] [--T 30] [--repeats 3]
"""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from trajopt_b200 import api, capi, problems  # noqa: E402


def solve(p, max_time):
    sqp = capi.default_sqp_params()
    sqp.max_time = max_time
    p.set_sqp_params(sqp)
    got = p.solve()
    B = p.desc.B
    start, ended = C.c_uint64(0), np.zeros(B, np.int32)
    p.lib.tb200_debug_time_limit(p.handle, C.byref(start), ended.ctypes.data_as(C.POINTER(C.c_int32)))
    sched = np.zeros(1 + 2 * B, np.uint64)
    p.lib.tb200_debug_schedule(p.handle, sched.ctypes.data_as(C.POINTER(C.c_uint64)))
    finish_ms = (sched[1:1 + B].astype(np.int64) - np.int64(start.value)) * 1e-6
    return got, ended, finish_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--T", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3, help="solves per budget (the table shows the median device time)")
    a = ap.parse_args()
    d = problems.config2(B=a.B, T=a.T)
    p = api.Problem(d)
    solve(p, sys.float_info.max)  # warm-up
    runs = [solve(p, sys.float_info.max) for _ in range(a.repeats)]
    t0 = float(np.median([g["timing"]["total_ms"] for g, _, _ in runs]))
    got = runs[0][0]
    print(f"configs[2] B={a.B} T={a.T}: no limit: {t0:.1f} ms, converged {(got['status'] == capi.OPT_CONVERGED).sum()}, "
          f"finish p50 {np.median(runs[0][2]):.1f} ms, last {runs[0][2].max():.1f} ms")
    print(f"{'budget':>7} {'max_time ms':>11} {'converged':>9} {'time limit':>10} {'ended by clock':>14} {'device ms':>9} "
          f"{'max overshoot ms':>16}")
    for f in (0.1, 0.25, 0.5, 0.75):
        limit_ms = f * t0
        runs = [solve(p, limit_ms * 1e-3) for _ in range(a.repeats)]
        ms = [g["timing"]["total_ms"] for g, _, _ in runs]
        k = int(np.argsort(ms)[len(ms) // 2])
        g, ended, fin = runs[k]
        over = max(float((fin - limit_ms).max()), 0.0)
        print(f"{f:7.2f} {limit_ms:11.1f} {(g['status'] == capi.OPT_CONVERGED).sum():9d} "
              f"{(g['status'] == capi.OPT_TIME_LIMIT).sum():10d} {ended.sum():14d} {ms[k]:9.1f} {over:16.2f}")
    p.close()


if __name__ == "__main__":
    main()
