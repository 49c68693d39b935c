// Look-up of the persistent SQP kernel instances (one translation unit each: solve_inst_<D>_<PAIR>.cu), generated from the
// joint-count lists of kernels.h.
#include <cuda_runtime.h>

#include "kernels.h"

namespace tb200 {
#define TB200_DECL(D, P)                  \
  SolveKernelFn solve_kernel_inst_##D##_##P(); \
  SolveKernelFn solve_kernel_sing_inst_##D##_##P(); \
  int qp_prof_inst_##D##_##P(unsigned long long*, int);
#define TB200_DECL_0(D) TB200_DECL(D, 0)
#define TB200_DECL_1(D) TB200_DECL(D, 1)
TB200_JOINT_COUNTS(TB200_DECL_0)
TB200_PAIR_JOINT_COUNTS(TB200_DECL_1)
#undef TB200_DECL_1
#undef TB200_DECL_0
#undef TB200_DECL

SolveKernelFn solve_kernel_for(int D, bool pair_rows, bool sing) {
#define TB200_PICK(DD, P) \
  if (D == DD && pair_rows == static_cast<bool>(P)) return sing ? solve_kernel_sing_inst_##DD##_##P() : solve_kernel_inst_##DD##_##P();
#define TB200_PICK_0(DD) TB200_PICK(DD, 0)
#define TB200_PICK_1(DD) TB200_PICK(DD, 1)
  TB200_JOINT_COUNTS(TB200_PICK_0)
  TB200_PAIR_JOINT_COUNTS(TB200_PICK_1)
#undef TB200_PICK_1
#undef TB200_PICK_0
#undef TB200_PICK
  return nullptr;
}
int qp_debug_prof(unsigned long long* out, int reset) {
  int rc = -1;
  if (!reset && out)
    for (int i = 0; i < kQpProfSlots; ++i) out[i] = 0;
#define TB200_PROF(D, P) \
  if (qp_prof_inst_##D##_##P(out, reset) == 0) rc = 0;
#define TB200_PROF_0(D) TB200_PROF(D, 0)
#define TB200_PROF_1(D) TB200_PROF(D, 1)
  TB200_JOINT_COUNTS(TB200_PROF_0)
  TB200_PAIR_JOINT_COUNTS(TB200_PROF_1)
#undef TB200_PROF_1
#undef TB200_PROF_0
#undef TB200_PROF
  return rc;
}
}  // namespace tb200
