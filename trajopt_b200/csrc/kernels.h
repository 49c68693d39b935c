// Kernel instances live in their own translation units (eval_inst_<D>[_sing].cu, solve_inst_<D>_<PAIR>[_sing].cu) so that
// they build in parallel; the host side of the C ABI (trajopt_b200.cu) reaches them through these look-ups
// (eval_kernels.cu, solve_kernels.cu).
#pragma once
#include "device_types.cuh"

// The joint counts with kernel instances: X(D) for each.  Both look-ups are generated from these lists, and every entry
// needs its units: eval_inst_<D>.cu, eval_inst_<D>_sing.cu, solve_inst_<D>_0.cu, solve_inst_<D>_0_sing.cu, and for the
// counts of the second list (QP rows that span two waypoints: CartVel, continuous collision) also
// solve_inst_<D>_1.cu and solve_inst_<D>_1_sing.cu.
#define TB200_JOINT_COUNTS(X) X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16)
#define TB200_PAIR_JOINT_COUNTS(X) X(2) X(7)

namespace tb200 {
struct EvalExtra;
struct SolveCtl;
using SolveKernelFn = void (*)(DevProblem, EvalExtra, SolveCtl);
using EvalKernelFn = void (*)(DevProblem, EvalExtra, int, const double*);
// The persistent SQP kernel (solve_kernel.cuh).  pair_rows: QP rows may span two consecutive waypoints (2*D
// coefficients per padded row instead of D); sing: the problem has AvoidSingularity objects (the instances without them
// carry none of the term's code).  nullptr: no instance for this number of joints.
SolveKernelFn solve_kernel_for(int D, bool pair_rows, bool sing);
EvalKernelFn eval_kernel_for(int D, bool sing);
int eval_debug_prof(unsigned long long* out, int reset);  // TB200_EVAL_PROFILE builds of an eval_inst_<D>.cu only
constexpr int kQpProfSlots = 32;  // phase counters of a TB200_PROFILE build (slot meanings: scripts/prof_phases.py)
int qp_debug_prof(unsigned long long* out, int reset);  // out[kQpProfSlots]; TB200_PROFILE builds only (else returns -1)
}  // namespace tb200
