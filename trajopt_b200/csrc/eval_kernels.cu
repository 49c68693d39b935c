// Instances of the convexify + exact evaluation + SQP decision kernel (eval_kernel.cuh), one per joint count.
#include <cuda_runtime.h>

#include "eval_kernel.cuh"
#include "kernels.h"

namespace tb200 {
EvalKernelFn eval_kernel_for(int D, bool sing) {
  switch (D) {
    case 2: return sing ? eval_convexify_decide_kernel<2, 1> : eval_convexify_decide_kernel<2>;
    case 3: return sing ? eval_convexify_decide_kernel<3, 1> : eval_convexify_decide_kernel<3>;
    case 6: return sing ? eval_convexify_decide_kernel<6, 1> : eval_convexify_decide_kernel<6>;
    case 7: return sing ? eval_convexify_decide_kernel<7, 1> : eval_convexify_decide_kernel<7>;
    case 14: return sing ? eval_convexify_decide_kernel<14, 1> : eval_convexify_decide_kernel<14>;
    default: return nullptr;
  }
}
int eval_debug_prof(unsigned long long* out, int reset) {
#ifdef TB200_EVAL_PROFILE
  if (reset == 2) {  // the per-CTA timeline of the last launch: out[3 * 4096]
    cudaMemcpyFromSymbol(out, g_eval_trace, sizeof(g_eval_trace));
    return 0;
  }
  if (reset) {
    unsigned long long z[16] = {0};
    cudaMemcpyToSymbol(g_eval_prof, z, sizeof(z));
    return 0;
  }
  cudaMemcpyFromSymbol(out, g_eval_prof, 16 * sizeof(unsigned long long));
  return 0;
#else
  (void)out; (void)reset;
  return -1;
#endif
}
}  // namespace tb200
