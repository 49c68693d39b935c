import sys, os, time, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
# needs a build of solve_kernels.cu with -DTB200_PROFILE, selected with TB200_LIB=<path to that .so>
from trajopt_b200 import api, problems
B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
cfg = sys.argv[2] if len(sys.argv) > 2 else "cfg2"
d = problems.CONFIGS[cfg](B=B, T={"cfg3": 50, "cfg4": 40}.get(cfg, 30))
p = api.Problem(d)
p.lib.tb200_debug_prof(None, 1)
t0 = time.time(); got = p.solve(); dt = time.time() - t0
prof = (C.c_ulonglong * 32)()  # kQpProfSlots
p.lib.tb200_debug_prof(prof, 0)
names = ["rows_coef", "scatter", "solve", "rows+vars", "-", "info+check", "factor(initial)", "scale", "qp_solve total", "launch-trajs", "iters-sum"]
tot_iters = got["n_admm_iters"].sum()
print(f"B={B} wall {dt:.2f}s, total ADMM iters {tot_iters}, qp solves {got['n_qp_solves'].sum()}, launches*trajs {prof[9]}")
for i, n in enumerate(names[:9]):
    print(f"  {n:22s} {prof[i]/1e6:10.1f} Mcycles  per-iter {prof[i]/max(tot_iters,1):9.0f} cycles")
nq = got['n_qp_solves'].sum()
# (slots 4, 14, 15, 9: every bcr_solve_sm, i.e. the polish passes' solves too; slot 9 then also counts the QP steps)
for slot, n in ((4, "solve: wait for the rhs barrier"), (14, "solve: level 0 down"), (15, "solve: upper levels down"), (9, "solve: upper levels up"),):
    print(f"  {n:32s} {prof[slot]/1e6:10.1f} Mcycles  per-iter {prof[slot]/max(tot_iters,1):9.0f} cycles")
print(f"  assemble (all calls) {prof[10]/1e6:10.1f} Mcycles, elimination (all calls) {prof[11]/1e6:10.1f} Mcycles")
# the parts of qp_solve outside the ADMM loop's hot phases, one slot each
for slot, n in ((5, "termination check (info_pass + check_termination)"), (22, "active-set guess hash (O1)"),
                (16, "polish: Z stash + set-up"), (23, "polish: factorisation"), (12, "polish: refinement passes"),
                (19, "recovery after a failed polish"), (20, "rho-update refactorisations"), (21, "ADMM block entry")):
    print(f"  {n:52s} {prof[slot]/1e6:10.1f} Mcycles  per-iter {prof[slot]/max(tot_iters,1):7.0f} cycles")
# slots 24 + 2 kind / 25 + 2 kind: assembly / elimination of assemble_factor per kind; 31 counts the calls of kind 1
print("  factorisations (assemble_factor), per kind: assembly | elimination")
for k, (n, calls) in enumerate((("initial", nq), ("rho update / recovery", prof[31]), ("polish", prof[13]))):
    a, e = prof[24 + 2 * k], prof[25 + 2 * k]
    print(f"  {n:24s} per-iter {a/max(tot_iters,1):7.0f} | {e/max(tot_iters,1):7.0f} cycles   "
          f"{calls} calls, per call {a/max(calls,1):8.0f} | {e/max(calls,1):8.0f} cycles")
print(f"  bcr_factor's block inversions (all calls) {prof[30]/1e6:10.1f} Mcycles")
print(f"  polishes {prof[13]} ({prof[13]/nq:.2f} per QP): early {prof[17]} ({prof[17]/nq:.2f} per QP), "
      f"final {prof[18]} ({prof[18]/nq:.2f} per QP)")
