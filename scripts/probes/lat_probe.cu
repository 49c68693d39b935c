// Latency probe for the building blocks of one ADMM iteration (one CTA of 256 threads on one SM):
// dependent DFMA chain, 64-bit shuffle, LDS.128, __syncthreads with 8 warps, and one block-cyclic-reduction level
// (7 x LDS.128 + 14 DFMA in two chains + shuffle + STS + barrier).  nvcc -arch=sm_90a -O3 lat_probe.cu -o lat_probe
#include <cstdio>
#include <cuda_runtime.h>

__global__ void probe(double* out, long long* cyc, int n) {
  __shared__ double2 sm2[2048];
  double* sm = reinterpret_cast<double*>(sm2);
  const int tid = threadIdx.x;
  for (int i = tid; i < 4096; i += blockDim.x) sm[i] = 1.0 + 1e-9 * i;
  __syncthreads();
  double a = 1.0 + tid * 1e-12, b = 0.999999, c = 1e-9;
  long long t0, t1;
  // 1. dependent DFMA chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < n; ++i) a = a * b + c;
  t1 = clock64();
  if (tid == 0) cyc[0] = t1 - t0;
  // 2. 64-bit shuffle chain
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < n; ++i) a += __shfl_xor_sync(0xffffffffu, a, 1);
  t1 = clock64();
  if (tid == 0) cyc[1] = t1 - t0;
  a = a * 1e-300 + 1.0;
  // 3. dependent LDS.64 chain (pointer chasing through indices)
  int idx = tid & 255;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < n; ++i) idx = (static_cast<int>(sm[idx]) + idx) & 4095;
  t1 = clock64();
  if (tid == 0) cyc[2] = t1 - t0;
  // 4. barrier only
  __syncthreads();
  t0 = clock64();
  for (int i = 0; i < n; ++i) __syncthreads();
  t1 = clock64();
  if (tid == 0) cyc[3] = t1 - t0;
  // 5. STS -> barrier -> LDS -> DFMA (a value handed to the neighbour thread every step)
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    sm[tid] = a;
    __syncthreads();
    a = sm[(tid + 33) & 255] * b + c;
    __syncthreads();
  }
  t1 = clock64();
  if (tid == 0) cyc[4] = t1 - t0;
  // 6. one BCR level: 7 x LDS.128 of the vector, 14 DFMA against register rows (two chains), shuffle, STS, barrier
  double m[14];
#pragma unroll
  for (int k = 0; k < 14; ++k) m[k] = 1e-3 * (k + 1) + 1e-6 * tid;
  double* v = sm + 1024;
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    const double2* y2 = reinterpret_cast<const double2*>(v + ((tid >> 1) / 14) * 28);
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const double2 yy = y2[k];
      a0 += m[2 * k] * yy.x;
      a1 += m[2 * k + 1] * yy.y;
    }
    double s = a0 + a1;
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if ((tid & 1) == 0) v[256 + (tid >> 1)] -= s * 1e-9;
    __syncthreads();
  }
  t1 = clock64();
  if (tid == 0) cyc[5] = t1 - t0;
  // 7. the same level executed by warp 0 only while the other warps go straight to the barrier
  t0 = clock64();
  for (int i = 0; i < n; ++i) {
    if (tid < 32) {
      const double2* y2 = reinterpret_cast<const double2*>(v + ((tid >> 1) / 14) * 28);
      double a0 = 0.0, a1 = 0.0;
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const double2 yy = y2[k];
        a0 += m[2 * k] * yy.x;
        a1 += m[2 * k + 1] * yy.y;
      }
      double s = a0 + a1;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if ((tid & 1) == 0) v[256 + (tid >> 1)] -= s * 1e-9;
    }
    __syncthreads();
  }
  t1 = clock64();
  if (tid == 0) cyc[6] = t1 - t0;
  // 8. named barrier among 2 warps (64 threads) with the same body
  t0 = clock64();
  if (tid < 64) {
    for (int i = 0; i < n; ++i) {
      const double2* y2 = reinterpret_cast<const double2*>(v + ((tid >> 1) / 14) * 28);
      double a0 = 0.0, a1 = 0.0;
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const double2 yy = y2[k];
        a0 += m[2 * k] * yy.x;
        a1 += m[2 * k + 1] * yy.y;
      }
      double s = a0 + a1;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if ((tid & 1) == 0) v[256 + (tid >> 1)] -= s * 1e-9;
      asm volatile("bar.sync 1, 64;" ::: "memory");
    }
  }
  t1 = clock64();
  if (tid == 0) cyc[7] = t1 - t0;
  // 9. warp-only variant: __syncwarp instead of a barrier
  t0 = clock64();
  if (tid < 32) {
    for (int i = 0; i < n; ++i) {
      const double2* y2 = reinterpret_cast<const double2*>(v + ((tid >> 1) / 14) * 28);
      double a0 = 0.0, a1 = 0.0;
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const double2 yy = y2[k];
        a0 += m[2 * k] * yy.x;
        a1 += m[2 * k + 1] * yy.y;
      }
      double s = a0 + a1;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if ((tid & 1) == 0) v[256 + (tid >> 1)] -= s * 1e-9;
      __syncwarp();
    }
  }
  t1 = clock64();
  if (tid == 0) cyc[8] = t1 - t0;
  __syncthreads();
  out[tid] = a + idx + sm[tid];
}

int main() {
  double* out;
  long long* cyc;
  cudaMalloc(&out, 256 * sizeof(double));
  cudaMalloc(&cyc, 16 * sizeof(long long));
  const int n = 2048;
  for (int rep = 0; rep < 2; ++rep) probe<<<1, 256>>>(out, cyc, n);
  long long h[16];
  cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
  const char* names[] = {"dependent DFMA", "64-bit shfl_xor + DADD", "dependent LDS.64 (+cvt, add)", "__syncthreads (8 warps)",
                         "STS -> bar -> LDS -> DFMA -> bar", "BCR level, all 8 warps + __syncthreads",
                         "BCR level, warp 0 works, 8 warps sync", "BCR level, 2 warps, bar.sync 1,64", "BCR level, 1 warp, __syncwarp"};
  for (int i = 0; i < 9; ++i) printf("%-44s %8.1f cycles per step\n", names[i], double(h[i]) / n);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
