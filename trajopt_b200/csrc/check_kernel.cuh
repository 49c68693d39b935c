// Trajectory collision check (tb200_check_trajectories, DESIGN.md section 4.6): every trajectory of a batch against the
// robot spheres and the obstacle spheres of its problem, with one result slot per waypoint (DISCRETE) or per step pair
// (LVS_DISCRETE, CONTINUOUS, LVS_CONTINUOUS).  What tesseract's checkTrajectory answers for the reference, restated for
// this project's sphere model and with the sub-trajectory rules of its own collision terms.
#pragma once
#include <cuda_runtime.h>

#include "device_types.cuh"

namespace tb200 {

constexpr int kCheckThreads = 256;
constexpr int kCheckWarps = kCheckThreads / 32;

struct CheckArgs {
  const DevSegment* segs;      // [S] (the host's folded segment table)
  const DevSphere* spheres;    // [L] in the description's order
  const double* obstacles;     // [B or 1][O][4]
  const double* x;             // [B][T][D]
  int B, T, D, S, L, O, obstacles_per_traj;
  int type;                    // TB200_COLL_*
  int n_slots;                 // T (DISCRETE) or T - 1
  double lvs, margin;
  double* slot_min;            // [B][n_slots] minimum signed distance (NaN: a non-finite distance)
  int* slot_contacts;          // [B][n_slots] (sphere, obstacle, sub-state | sub-segment) triples closer than margin
  int* slot_argmin;            // [B][n_slots][3] sphere, obstacle, sub-index of the minimum (-1 when there is none)
  int* in_collision;           // [B]
  int* first_slot;             // [B] first slot with a contact, -1 if none
  double* min_distance;        // [B]
};

// Shared memory of one CTA, in doubles: the robot tables, then per warp the frames of one state, the sphere centres at
// the two ends of the running sub-segment and one joint vector.
__host__ __device__ inline int check_warp_doubles(int S, int L) { return S * 12 + 6 * L + kMaxDof; }
__host__ __device__ inline int check_smem_doubles(int S, int L) {
  return S * static_cast<int>(sizeof(DevSegment) / 8) + L * static_cast<int>(sizeof(DevSphere) / 8) +
         kCheckWarps * check_warp_doubles(S, L);
}

// Signed distance between an obstacle sphere ob = (x, y, z, r) and the robot sphere of radius r whose centre moves on
// the chord ca -> cb: the closest point of the chord (parameter clamped to [0, 1]) against the obstacle's centre.  ca ==
// cb is the sphere/sphere distance.  At parameter 1 the point is cb itself rather than ca + (cb - ca), so the state two
// sub-segments share gives both of them the same distance and the lower sub-index wins the tie.  (The convexify kernel
// keeps ca + s (cb - ca) for its rows: they stay bit for bit those of the oracle's CastCollisionEval.)
__device__ __forceinline__ double swept_sphere_distance(const double* ca, const double* cb, double r, const double4& ob) {
  const double wx = cb[0] - ca[0], wy = cb[1] - ca[1], wz = cb[2] - ca[2];
  const double ww = wx * wx + wy * wy + wz * wz;
  const double wd = (ob.x - ca[0]) * wx + (ob.y - ca[1]) * wy + (ob.z - ca[2]) * wz;
  double s = (ww > 0.0) ? wd / ww : 0.0;
  s = s < 0.0 ? 0.0 : (s > 1.0 ? 1.0 : s);
  const double px = s == 1.0 ? cb[0] : ca[0] + s * wx, py = s == 1.0 ? cb[1] : ca[1] + s * wy,
               pz = s == 1.0 ? cb[2] : ca[2] + s * wz;
  const double dx = ob.x - px, dy = ob.y - py, dz = ob.z - pz;
  return sqrt(dx * dx + dy * dy + dz * dz) - r - ob.w;
}

// Launches the slot kernel (one warp per (trajectory, slot)) and the per-trajectory summary on `st`.
cudaError_t launch_check_trajectories(const CheckArgs& a, int n_sm, cudaStream_t st);

}  // namespace tb200
