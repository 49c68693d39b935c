// Look-up of the convexify + exact evaluation + SQP decision kernel instances (one translation unit each:
// eval_inst_<D>[_sing].cu), generated from the joint-count list of kernels.h.
#include <cuda_runtime.h>

#include "kernels.h"

namespace tb200 {
#define TB200_DECL(D)                  \
  EvalKernelFn eval_kernel_inst_##D(); \
  EvalKernelFn eval_kernel_sing_inst_##D(); \
  int eval_prof_inst_##D(unsigned long long*, int);
TB200_JOINT_COUNTS(TB200_DECL)
#undef TB200_DECL

EvalKernelFn eval_kernel_for(int D, bool sing) {
#define TB200_PICK(DD) \
  if (D == DD) return sing ? eval_kernel_sing_inst_##DD() : eval_kernel_inst_##DD();
  TB200_JOINT_COUNTS(TB200_PICK)
#undef TB200_PICK
  return nullptr;
}
int eval_debug_prof(unsigned long long* out, int reset) {
  int rc = -1;
  if (!reset && out)
    for (int i = 0; i < 16; ++i) out[i] = 0;
#define TB200_PROF(D) \
  if (eval_prof_inst_##D(out, reset) == 0) rc = 0;
  TB200_JOINT_COUNTS(TB200_PROF)
#undef TB200_PROF
  return rc;
}
}  // namespace tb200
