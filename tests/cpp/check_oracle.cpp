// CPU model of the trajectory collision check (tb200_check_trajectories, DESIGN.md section 4.6), for
// tests/test_check_trajectories.py.  It restates the check with the oracle's robot model (oracle::Robot::fk) and the
// sub-trajectory rules of its CastCollisionEval (n = ceil(|q1 - q0| / lvs) sub-segments, states q0 + (q1 - q0) i/n with
// the waypoints themselves at i = 0 and i = n): a discrete test at each state or a swept test (capsule / sphere) over
// each sub-segment, over every (sphere, obstacle) candidate.  Built by the test and linked against liboracle.so; the
// oracle itself is left as it is.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>

#include "trajopt.hpp"

using namespace oracle;

namespace {
// closest point of the chord ca -> cb to the obstacle's centre; at parameter 1 the point is cb itself (the state two
// sub-segments share gives both the same distance)
double sweptSphereDistance(const double* ca, const double* cb, double r, const double* ob) {
  double w[3], ww = 0, wd = 0;
  for (int k = 0; k < 3; ++k) {
    w[k] = cb[k] - ca[k];
    ww += w[k] * w[k];
    wd += (ob[k] - ca[k]) * w[k];
  }
  double s = (ww > 0) ? wd / ww : 0.0;
  s = s < 0 ? 0.0 : (s > 1 ? 1.0 : s);
  double d2 = 0;
  for (int k = 0; k < 3; ++k) {
    const double d = ob[k] - (s == 1.0 ? cb[k] : ca[k] + s * w[k]);
    d2 += d * d;
  }
  return std::sqrt(d2) - r - ob[3];
}

// One trajectory x [T*D] against obstacles [O][4].  Per slot (T for DISCRETE, else T-1): minimum signed distance
// (NaN: non-finite), contacts, argmin (sphere, obstacle, sub-index; -1 when none).
void checkTrajectory(const Robot& robot, const double* obstacles, int O, const double* x, int T, int type, double lvs,
                     double margin, double* slot_min, int* slot_contacts, int* slot_argmin) {
  const int D = robot.n_dof, L = static_cast<int>(robot.spheres.size());
  const bool discrete = type == TB200_COLL_DISCRETE, swept = type == TB200_COLL_CONTINUOUS || type == TB200_COLL_LVS_CONTINUOUS;
  const bool sub = type == TB200_COLL_LVS_DISCRETE || type == TB200_COLL_LVS_CONTINUOUS;
  const int S = discrete ? T : T - 1;
  std::vector<Pose> fr;
  Vec u(D);
  // centres of every sphere at state i of n between q0 and q1
  auto centres = [&](const double* q0, const double* q1, int i, int n, Vec& c) {
    for (int j = 0; j < D; ++j) u[j] = (i == 0) ? q0[j] : (i == n ? q1[j] : q0[j] + (q1[j] - q0[j]) * (static_cast<double>(i) / n));
    robot.fk(u.data(), fr);
    c.resize(3 * L);
    for (int s = 0; s < L; ++s) {
      const tb200_sphere& sp = robot.spheres[s];
      const Pose& f = fr[sp.segment];
      for (int k = 0; k < 3; ++k)
        c[3 * s + k] = f.R[k * 3] * sp.center[0] + f.R[k * 3 + 1] * sp.center[1] + f.R[k * 3 + 2] * sp.center[2] + f.p[k];
    }
  };
  for (int t = 0; t < S; ++t) {
    const double* q0 = x + static_cast<size_t>(t) * D;
    const double* q1 = discrete ? q0 : q0 + D;
    int n = 1;
    if (sub) {
      double d2 = 0;
      for (int j = 0; j < D; ++j) d2 += (q1[j] - q0[j]) * (q1[j] - q0[j]);
      const double qd = std::sqrt(d2);
      if (std::isfinite(qd) && qd > lvs) {  // (a step of non-finite length is one sub-segment)
        const double nn = std::ceil(qd / lvs);
        n = nn >= static_cast<double>(std::numeric_limits<int>::max()) ? std::numeric_limits<int>::max() : static_cast<int>(nn);
      }
    }
    const int n_tests = discrete ? 1 : (swept ? n : n + 1);
    double best = std::numeric_limits<double>::infinity();  // non-finite distances rank as -inf
    int arg[3] = {-1, -1, -1};
    long long contacts = 0;
    if (L > 0 && O > 0) {
      std::vector<Vec> cen(swept ? n + 1 : n_tests);  // centres at the states 0..n (DISCRETE: the waypoint)
      for (size_t i = 0; i < cen.size(); ++i) centres(q0, q1, static_cast<int>(i), n, cen[i]);
      // (sphere, obstacle, sub) order: a later candidate replaces the best only when it is strictly smaller
      for (int s = 0; s < L; ++s)
        for (int o = 0; o < O; ++o)
          for (int i = 0; i < n_tests; ++i) {
            const double* pa = cen[i].data() + 3 * s;
            const double* pb = swept ? cen[i + 1].data() + 3 * s : pa;
            const double d = sweptSphereDistance(pa, pb, robot.spheres[s].radius, obstacles + 4 * o);
            const double v = std::isfinite(d) ? d : -std::numeric_limits<double>::infinity();
            if (v < best) {
              best = v;
              arg[0] = s; arg[1] = o; arg[2] = i;
            }
            contacts += !(std::isfinite(d) && d >= margin);
          }
    }
    slot_min[t] = (best == -std::numeric_limits<double>::infinity()) ? std::numeric_limits<double>::quiet_NaN() : best;
    slot_contacts[t] = contacts > std::numeric_limits<int>::max() ? std::numeric_limits<int>::max() : static_cast<int>(contacts);
    for (int k = 0; k < 3; ++k) slot_argmin[3 * t + k] = arg[k];
  }
}
}  // namespace

extern "C" {

// Trajectory collision check (tb200_check_trajectories) of x [B][T][D] against the description's robot and obstacles,
// trajectories [b0, b1).  Per slot (S = T for DISCRETE, else T - 1): slot_min [B][S], contacts [B][S], argmin [B][S][3];
// per trajectory: in_collision, first_slot, min_distance (derived from the slots).
int check_oracle_trajectories(const tb200_problem_desc* desc, int b0, int b1, const double* x, int type, double lvs,
                              double margin, double* slot_min, int32_t* contacts, int32_t* argmin, int32_t* in_collision,
                              int32_t* first_slot, double* min_distance) {
  const int T = desc->n_steps, D = desc->robot.n_dof, O = desc->n_obstacles;
  const int S = (type == TB200_COLL_DISCRETE) ? T : T - 1;
  const Robot robot(desc->robot);
#pragma omp parallel for schedule(dynamic)
  for (int b = b0; b < b1; ++b) {
    const double* obst = desc->obstacles ? desc->obstacles + (desc->obstacles_per_traj ? static_cast<size_t>(b) * O * 4 : 0) : nullptr;
    double* mn = slot_min + static_cast<size_t>(b) * S;
    int32_t* ct = contacts + static_cast<size_t>(b) * S;
    checkTrajectory(robot, obst, obst ? O : 0, x + static_cast<size_t>(b) * T * D, T, type, lvs, margin, mn, ct,
                    argmin + static_cast<size_t>(b) * S * 3);
    int first = -1;
    bool nan = false;
    double m = std::numeric_limits<double>::infinity();
    for (int s = 0; s < S; ++s) {
      if (ct[s] > 0 && first < 0) first = s;
      nan = nan || std::isnan(mn[s]);
      m = std::min(m, mn[s]);
    }
    in_collision[b] = first >= 0;
    first_slot[b] = first;
    min_distance[b] = nan ? std::numeric_limits<double>::quiet_NaN() : m;
  }
  return 0;
}

}  // extern "C"
