// Trajectory collision check kernels (check_kernel.cuh).  One warp per (trajectory, slot), grid-stride: the warp walks
// the slot's states (a waypoint, or the sub-trajectory of a step pair) one at a time, runs the FK of each state
// cooperatively, and its lanes split the L * O (robot sphere, obstacle) candidates of every state or sub-segment.
#include <math_constants.h>

#include <climits>

#include "../../include/trajopt_b200.h"
#include "check_kernel.cuh"
#include "eval_kernel.cuh"  // cp_async8

namespace tb200 {
namespace {

// FK of one joint state by a warp, from a segment table in shared memory: local frames with the lanes over the segments,
// then the chain products row by row (lanes 0-2).  F: [Sg][12] world frames (R row-major, p).  The same products as
// warp_fk of the evaluation kernel, which reads the table through its DevProblem (routing that one through a pointer
// changes the code of the persistent solve kernels).
__device__ void check_warp_fk(const DevSegment* segs, int Sg, const double* q, double* F, int lane) {
  for (int sg = lane; sg < Sg; sg += 32) {
    const DevSegment& g = segs[sg];
    Frame loc;
    segment_local_q(g, g.q_index >= 0 ? q[g.q_index] : 0.0, loc);
    double* f = F + sg * 12;
    for (int i = 0; i < 9; ++i) f[i] = loc.R[i];
    for (int i = 0; i < 3; ++i) f[9 + i] = loc.p[i];
  }
  __syncwarp();
  const int i = lane < 3 ? lane : 0;
  for (int sg = 0; sg < Sg; ++sg) {
    const int parent = segs[sg].parent;
    double l[12];
    for (int k = 0; k < 12; ++k) l[k] = F[sg * 12 + k];
    __syncwarp();  // every row has read the local frame before it is overwritten
    if (lane < 3 && parent >= 0) {
      const double* P = F + parent * 12;
      const double r0 = P[i * 3], r1 = P[i * 3 + 1], r2 = P[i * 3 + 2], pi = P[9 + i];
      F[sg * 12 + i * 3 + 0] = r0 * l[0] + r1 * l[3] + r2 * l[6];
      F[sg * 12 + i * 3 + 1] = r0 * l[1] + r1 * l[4] + r2 * l[7];
      F[sg * 12 + i * 3 + 2] = r0 * l[2] + r1 * l[5] + r2 * l[8];
      F[sg * 12 + 9 + i] = r0 * l[9] + r1 * l[10] + r2 * l[11] + pi;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kCheckThreads) check_trajectories_kernel(const __grid_constant__ CheckArgs a) {
  extern __shared__ double sm[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int SD = static_cast<int>(sizeof(DevSegment) / 8), PD = static_cast<int>(sizeof(DevSphere) / 8);
  // the robot tables, once per CTA
  for (int i = tid; i < a.S * SD; i += kCheckThreads) cp_async8(sm + i, reinterpret_cast<const double*>(a.segs) + i);
  for (int i = tid; i < a.L * PD; i += kCheckThreads) cp_async8(sm + a.S * SD + i, reinterpret_cast<const double*>(a.spheres) + i);
  cp_async_wait_all();
  __syncthreads();
  const DevSegment* segs = reinterpret_cast<const DevSegment*>(sm);
  const DevSphere* sphs = reinterpret_cast<const DevSphere*>(sm + a.S * SD);
  double* F = sm + a.S * SD + a.L * PD + warp * check_warp_doubles(a.S, a.L);  // this warp's frames of one state
  double* cen0 = F + a.S * 12;                                                 // [L][3] centres, two states
  double* cen1 = cen0 + 3 * a.L;
  double* qv = cen1 + 3 * a.L;                                                  // [D] the state
  const int T = a.T, D = a.D, L = a.L, O = a.O, LO = L * O, ns = a.n_slots;
  const bool swept = a.type == TB200_COLL_CONTINUOUS || a.type == TB200_COLL_LVS_CONTINUOUS;
  const bool lvs = a.type == TB200_COLL_LVS_DISCRETE || a.type == TB200_COLL_LVS_CONTINUOUS;
  const long long items = static_cast<long long>(a.B) * ns;
  for (long long it = static_cast<long long>(blockIdx.x) * kCheckWarps + warp; it < items;
       it += static_cast<long long>(gridDim.x) * kCheckWarps) {
    const int b = static_cast<int>(it / ns), s = static_cast<int>(it - static_cast<long long>(b) * ns);
    const double* q0 = a.x + (static_cast<size_t>(b) * T + s) * D;
    const double* q1 = (a.type == TB200_COLL_DISCRETE) ? q0 : q0 + D;
    const double* obst = a.obstacles + (a.obstacles_per_traj ? static_cast<size_t>(b) * O * 4 : 0);
    // n sub-segments of the pair: ceil(|q1 - q0| / lvs), 1 when the step is no longer than lvs.  A step of non-finite
    // length is one sub-segment (its distances are non-finite and count as contacts); above INT_MAX it is clamped.
    int n = 1;
    if (lvs) {
      double d2 = 0.0;
      for (int j = 0; j < D; ++j) d2 += (q1[j] - q0[j]) * (q1[j] - q0[j]);
      const double qd = sqrt(d2);
      if (isfinite(qd) && qd > a.lvs) {
        const double nn = ceil(qd / a.lvs);
        n = nn >= static_cast<double>(INT_MAX) ? INT_MAX : static_cast<int>(nn);
      }
    }
    // the tests of the slot: discrete ones at the states 0..n (DISCRETE: the waypoint alone), swept ones over the
    // sub-segments 0..n-1
    const int n_tests = (a.type == TB200_COLL_DISCRETE) ? 1 : (swept ? n : n + 1);
    // centres of every robot sphere at state i of the pair (i = 0 and i = n: the waypoints themselves)
    auto centres_at = [&](int i, double* dst) {
      if (lane < D) {
        const double u0 = q0[lane], u1 = q1[lane];
        qv[lane] = (i == 0) ? u0 : (i == n ? u1 : u0 + (u1 - u0) * (static_cast<double>(i) / n));
      }
      __syncwarp();
      check_warp_fk(segs, a.S, qv, F, lane);
      for (int w = lane; w < L; w += 32) {
        const DevSphere& sp = sphs[w];
        const double* f = F + sp.segment * 12;
        for (int k = 0; k < 3; ++k)
          dst[w * 3 + k] = f[k * 3] * sp.c[0] + f[k * 3 + 1] * sp.c[1] + f[k * 3 + 2] * sp.c[2] + f[9 + k];
      }
      __syncwarp();
    };
    // per lane: the smallest (distance, key) it has seen, key = candidate << 32 | sub-index ((sphere, obstacle, sub)
    // order); a non-finite distance ranks below every finite one
    double best = CUDART_INF;
    unsigned long long best_key = ~0ull;
    long long contacts = 0;  // (warp-uniform)
    double* ca = cen0;
    double* cb = cen1;
    if (LO > 0) {
      centres_at(0, ca);
      for (int i = 0; i < n_tests; ++i) {
        if (swept) centres_at(i + 1, cb);
        else if (i > 0) centres_at(i, ca);
        const double* cend = swept ? cb : ca;
        for (int c0 = 0; c0 < LO; c0 += 32) {
          const int pr = c0 + lane;
          bool contact = false;
          if (pr < LO) {
            const int sl = pr / O, o = pr - sl * O;
            const double4 ob = *reinterpret_cast<const double4*>(obst + o * 4);
            const double d = swept_sphere_distance(ca + sl * 3, cend + sl * 3, sphs[sl].r, ob);
            const bool finite = isfinite(d);
            const double v = finite ? d : -CUDART_INF;
            const unsigned long long key = (static_cast<unsigned long long>(pr) << 32) | static_cast<unsigned>(i);
            if (v < best || (v == best && key < best_key)) {
              best = v;
              best_key = key;
            }
            contact = !(finite && d >= a.margin);
          }
          contacts += __popc(__ballot_sync(0xffffffffu, contact));
        }
        if (swept) {  // the end of this sub-segment starts the next
          double* t = ca;
          ca = cb;
          cb = t;
        }
      }
    }
    for (int off = 16; off > 0; off >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, best, off);
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, best_key, off);
      if (ov < best || (ov == best && ok < best_key)) {
        best = ov;
        best_key = ok;
      }
    }
    if (lane == 0) {
      const size_t o = static_cast<size_t>(b) * ns + s;
      const bool found = best_key != ~0ull;
      const int pr = found ? static_cast<int>(best_key >> 32) : -1;
      a.slot_min[o] = (best == -CUDART_INF) ? CUDART_NAN : best;
      a.slot_contacts[o] = contacts > INT_MAX ? INT_MAX : static_cast<int>(contacts);
      a.slot_argmin[3 * o] = found ? pr / O : -1;
      a.slot_argmin[3 * o + 1] = found ? pr % O : -1;
      a.slot_argmin[3 * o + 2] = found ? static_cast<int>(best_key & 0xffffffffu) : -1;
    }
    __syncwarp();  // the frames and centres are reused by the warp's next item
  }
}

// Per trajectory, from its slots: in collision, the first slot with a contact and the minimum distance (NaN when a slot
// has one).  One warp per trajectory.
__global__ void check_summary_kernel(const __grid_constant__ CheckArgs a) {
  const int lane = threadIdx.x & 31;
  const int b = static_cast<int>((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (b >= a.B) return;  // (whole warps)
  int first = INT_MAX;
  double mn = CUDART_INF;
  bool nan = false;
  for (int s = lane; s < a.n_slots; s += 32) {
    const size_t o = static_cast<size_t>(b) * a.n_slots + s;
    if (a.slot_contacts[o] > 0 && s < first) first = s;
    const double v = a.slot_min[o];
    nan = nan || v != v;
    mn = fmin(mn, v);
  }
  for (int off = 16; off > 0; off >>= 1) {
    first = min(first, __shfl_xor_sync(0xffffffffu, first, off));
    mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, off));
  }
  nan = __any_sync(0xffffffffu, nan);
  if (lane == 0) {
    a.in_collision[b] = first != INT_MAX;
    a.first_slot[b] = first == INT_MAX ? -1 : first;
    a.min_distance[b] = nan ? CUDART_NAN : mn;
  }
}

}  // namespace

cudaError_t launch_check_trajectories(const CheckArgs& a, int n_sm, cudaStream_t st) {
  const long long items = static_cast<long long>(a.B) * a.n_slots;
  if (items > 0) {
    const size_t smem = static_cast<size_t>(check_smem_doubles(a.S, a.L)) * sizeof(double);
    cudaError_t e = cudaFuncSetAttribute(check_trajectories_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, check_trajectories_kernel, kCheckThreads, smem);
    if (e != cudaSuccess) return e;
    const long long want = (items + kCheckWarps - 1) / kCheckWarps;
    const long long cap = static_cast<long long>(per_sm > 0 ? per_sm : 1) * n_sm;
    check_trajectories_kernel<<<static_cast<int>(want < cap ? want : cap), kCheckThreads, smem, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  check_summary_kernel<<<(a.B + 3) / 4, 128, 0, st>>>(a);
  return cudaGetLastError();
}

}  // namespace tb200
