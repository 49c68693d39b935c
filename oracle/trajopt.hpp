// ORACLE — TEST INFRASTRUCTURE ONLY (see sco.hpp).  CPU fp64 restatement of the reference's
// trajopt term library for the hot path, written from scratch:
//   * joint-space terms     trajopt/src/trajectory_costs.cpp:12-754
//   * CartPose / CartVel    trajopt/src/kinematic_terms.cpp:187-425
//   * collision terms       trajopt/src/collision_terms.cpp:203-383, 540-556, 655-691, 1283-1412
//   * problem assembly      trajopt/src/problem_description.cpp:410-542, 553-592, 901-987, 1011-1057,
//                           1078-1176, 1197-1372, 1393-1493, 1714-1837
// Kinematics and the Cartesian error helpers live in tesseract (not in the reference tree):
// JointGroup::calcFwdKin / calcJacobian, tesseract::common::calcTransformError /
// calcJacobianTransformErrorDiff / jacobianChangeRefPoint are restated from their published
// behaviour [EXT]; they are pinned through the reference's own tests that exercise them
// (analytic-vs-numeric Jacobian agreement kinematic_costs_unit.cpp:60-97, the self-consistent IK
// test cart_position_optimization_unit.cpp:99-135, numerical_ik_unit.cpp:60-124).
// Collision geometry is sphere/sphere closed form (SURVEY.md §8d) — Bullet contact output is
// "parity unpinned" in the reference itself (only in-collision -> collision-free booleans).
#pragma once
#include "../include/trajopt_b200.h"
#include "sco.hpp"

namespace oracle {

struct Pose {
  double R[9];  // row-major
  double p[3];
};
Pose poseIdentity();
Pose poseMul(const Pose& a, const Pose& b);
Pose poseInv(const Pose& a);
Pose poseFromXyzWxyz(const double* xyz, const double* wxyz);
void rotToQuatWxyz(const double* R, double* wxyz);
// tesseract::common::calcRotationalError [EXT]: axis*angle with angle in [-pi, pi]
void calcRotationalError(const double* R, double out[3]);
// tesseract::common::calcTransformError(t1, t2) [EXT]: error of t1^-1 * t2
void calcTransformError(const Pose& t1, const Pose& t2, double out[6]);
// tesseract::common::calcJacobianTransformErrorDiff(target, source, source_perturbed) [EXT]
void calcJacobianTransformErrorDiff(const Pose& target, const Pose& source, const Pose& source_pert, double out[6]);

struct Robot {
  int n_dof = 0;
  std::vector<tb200_segment> segs;
  std::vector<tb200_sphere> spheres;
  Vec lower, upper;
  explicit Robot(const tb200_robot& r);
  void fk(const double* q, std::vector<Pose>& frames) const;  // frame of every segment, scene-root frame
  // 6 x n_dof geometric Jacobian of segment `link` at world point `point` (row-major J[6][n_dof]):
  // JointGroup::calcJacobian + jacobianChangeRefPoint [EXT]
  void jacobian(const std::vector<Pose>& frames, int link, const double* point, std::vector<Vec>& J) const;
};

struct TrajProblem {
  std::shared_ptr<OptProb> prob;
  std::shared_ptr<Robot> robot;
  int T = 0, D = 0;
  Vec init;  // [T*D]
  std::vector<std::string> cost_names, cnt_names;
  // Hooks for the kernel-level parity tests (fixed dense layout shared with the CUDA path):
  // coefficient-scaled Cartesian error rows (err, jac rows over the term's variables), in term order;
  std::vector<std::function<void(const Vec& x, Vec& err, std::vector<Vec>& jac)>> cart_hooks;
  // dense candidate collision rows [(sphere, obstacle)] = {grad[D], dist0, margin, coeff or 0 if filtered}: the cost
  // objects' first, then the constraints', each in term order
  std::vector<std::function<void(const Vec& x, std::vector<Vec>& rows)>> coll_hooks;
};
// avoid_singularity: J [6][D] row-major -> its smallest singular value and singular vectors u[6], v[D] (the undefined
// one of the pair is 0 when sigma is 0); the geometric Jacobian [6][D] of the link's origin at q; err and the
// unscaled gradient of one waypoint (any output may be NULL)
namespace sing {
void jacobiSvdMin(const double* J, int D, double& sigma, double* u, double* v);
void jacobianAt(const Robot& robot, const double* q, int link, std::vector<double>& J);
void errGrad(const Robot& robot, const double* q, int link, double lambda, double* err, double* grad, double* sigma_out);
}  // namespace sing

// One trajectory `b` of the batched description -> the reference's TrajOptProb
// (ConstructProblem, problem_description.cpp:410-542).
// cast_cap: rows per step pair of the continuous collision evaluator's fixed-layout output (< 0: compute it,
// tb200inl_cast_rows_per_pair)
TrajProblem buildProblem(const tb200_problem_desc& desc, int b, int cast_cap = -1);
SQPParams sqpParamsFrom(const tb200_sqp_params& p);
QPSettings qpSettingsFrom(const tb200_qp_settings& s);

}  // namespace oracle
