// Kernel instances live in their own translation units (eval_kernels.cu, solve_kernels.cu, solve_kernels_pair.cu) so that they build in
// parallel; the host side of the C ABI (trajopt_b200.cu) reaches them through these look-ups.
#pragma once
#include "device_types.cuh"

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
int eval_debug_prof(unsigned long long* out, int reset);  // TB200_EVAL_PROFILE builds of eval_kernels.cu only
constexpr int kQpProfSlots = 32;  // phase counters of a TB200_PROFILE build (slot meanings: scripts/prof_phases.py)
int qp_debug_prof(unsigned long long* out, int reset);  // out[kQpProfSlots]; TB200_PROFILE builds only (else returns -1)
}  // namespace tb200
