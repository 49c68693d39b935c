// One instance of the convexify + exact evaluation + SQP decision kernel (eval_kernel.cuh) per translation unit, so that
// the instances build side by side: the including .cu defines TB200_INST_D (joints) and TB200_INST_SING 1 for the
// instance of problems with AvoidSingularity objects.
#include <cuda_runtime.h>

#include "eval_kernel.cuh"
#include "kernels.h"

#define TB200_CAT2_(a, b) a##b
#define TB200_CAT2(a, b) TB200_CAT2_(a, b)

namespace tb200 {
#if TB200_INST_SING
EvalKernelFn TB200_CAT2(eval_kernel_sing_inst_, TB200_INST_D)() { return eval_convexify_decide_kernel<TB200_INST_D, 1>; }
#else
EvalKernelFn TB200_CAT2(eval_kernel_inst_, TB200_INST_D)() { return eval_convexify_decide_kernel<TB200_INST_D>; }
// TB200_EVAL_PROFILE builds: the cycle stamps of this translation unit (else -1).  reset 0: add the counters to out[16];
// 1: clear them; 2: the per-CTA timeline of the last launch into out[3 * 4096]
int TB200_CAT2(eval_prof_inst_, TB200_INST_D)(unsigned long long* out, int reset) {
#ifdef TB200_EVAL_PROFILE
  if (reset == 2) {
    cudaMemcpyFromSymbol(out, g_eval_trace, sizeof(g_eval_trace));
    return 0;
  }
  if (reset) {
    unsigned long long z[16] = {0};
    cudaMemcpyToSymbol(g_eval_prof, z, sizeof(z));
    return 0;
  }
  unsigned long long t[16];
  cudaMemcpyFromSymbol(t, g_eval_prof, sizeof(t));
  for (int i = 0; i < 16; ++i) out[i] += t[i];
  return 0;
#else
  (void)out;
  (void)reset;
  return -1;
#endif
}
#endif
}  // namespace tb200
