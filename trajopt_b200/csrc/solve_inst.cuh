// One instance of the persistent SQP kernel (solve_kernel.cuh) per translation unit, so that the instances build side by
// side: the including .cu defines TB200_INST_D (joints; the block size of the block-cyclic-reduction factor is 2*D)
// and TB200_INST_PAIR (1: QP rows may span two consecutive waypoints — CartVel, continuous collision), and
// TB200_INST_SING 1 for the instance of problems with AvoidSingularity objects.
#include <cuda_runtime.h>

#include "solve_kernel.cuh"
#include "kernels.h"

#define TB200_CAT3_(a, b, c) a##b##_##c
#define TB200_CAT3(a, b, c) TB200_CAT3_(a, b, c)

namespace tb200 {
#if TB200_INST_SING
SolveKernelFn TB200_CAT3(solve_kernel_sing_inst_, TB200_INST_D, TB200_INST_PAIR)() {
  return solve_kernel<TB200_INST_D, TB200_INST_PAIR, 1>;
}
#else
SolveKernelFn TB200_CAT3(solve_kernel_inst_, TB200_INST_D, TB200_INST_PAIR)() {
  return solve_kernel<TB200_INST_D, TB200_INST_PAIR>;
}
// TB200_PROFILE builds: the phase counters of this translation unit (else -1)
int TB200_CAT3(qp_prof_inst_, TB200_INST_D, TB200_INST_PAIR)(unsigned long long* out, int reset) {
#ifdef TB200_PROFILE
  static_assert(sizeof(g_prof) == kQpProfSlots * sizeof(unsigned long long), "g_prof and kQpProfSlots disagree");
  if (reset) {
    unsigned long long z[kQpProfSlots] = {0};
    cudaMemcpyToSymbol(g_prof, z, sizeof(z));
    return 0;
  }
  unsigned long long t[kQpProfSlots];
  cudaMemcpyFromSymbol(t, g_prof, sizeof(t));
  for (int i = 0; i < kQpProfSlots; ++i) out[i] += t[i];
  return 0;
#else
  (void)out;
  (void)reset;
  return -1;
#endif
}
#endif
}  // namespace tb200
