// Look-up of the persistent SQP kernel instances (one translation unit each: solve_inst_<D>_<PAIR>.cu).
#include <cuda_runtime.h>

#include "kernels.h"

namespace tb200 {
#define TB200_INSTANCES(X) X(2, 0) X(3, 0) X(6, 0) X(7, 0) X(14, 0) X(2, 1) X(7, 1)
#define TB200_DECL(D, P)                  \
  SolveKernelFn solve_kernel_inst_##D##_##P(); \
  SolveKernelFn solve_kernel_sing_inst_##D##_##P(); \
  int qp_prof_inst_##D##_##P(unsigned long long*, int);
TB200_INSTANCES(TB200_DECL)
#undef TB200_DECL

SolveKernelFn solve_kernel_for(int D, bool pair_rows, bool sing) {
#define TB200_PICK(DD, P) \
  if (D == DD && pair_rows == static_cast<bool>(P)) return sing ? solve_kernel_sing_inst_##DD##_##P() : solve_kernel_inst_##DD##_##P();
  TB200_INSTANCES(TB200_PICK)
#undef TB200_PICK
  return nullptr;
}
int qp_debug_prof(unsigned long long* out, int reset) {
  int rc = -1;
  if (!reset && out)
    for (int i = 0; i < kQpProfSlots; ++i) out[i] = 0;
#define TB200_PROF(D, P) \
  if (qp_prof_inst_##D##_##P(out, reset) == 0) rc = 0;
  TB200_INSTANCES(TB200_PROF)
#undef TB200_PROF
  return rc;
}
}  // namespace tb200
