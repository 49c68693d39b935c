// trajopt_b200.hpp — C++ host layer over the C ABI (trajopt_b200.h) under the reference's own names.
//
// The reference is a C++ library; what a caller writes against it for this path is
//   trajopt::ProblemConstructionInfo pci(env);  pci.basic_info...;  pci.cost_infos.push_back(term);  ...
//   auto prob = trajopt::ConstructProblem(pci);                      problem_description.hpp:235-259, 661
//   sco::BasicTrustRegionSQP opt(prob);  opt.setParameters(pci.opt_info);  opt.optimize();  opt.results();
// (trajopt/include/trajopt/problem_description.hpp:123-259, 273-659; trajopt_sco/include/trajopt_sco/optimizers.hpp:25-135).
// This header mirrors those types field by field for the terms the device path implements, for a BATCH of problems
// that share the robot, the term structure and the parameters (what differs per trajectory: initial trajectory,
// Cartesian targets, obstacle set), and flattens them into the POD description of the C ABI.  Differences from the
// reference, all forced by the missing tesseract / Eigen / jsoncpp dependencies (SURVEY.md section 8c):
//   * kinematics come as a RobotModel (URDF joint origins / axes / limits + link collision spheres) instead of a
//     tesseract::environment::Environment; frames are named links of that model;
//   * Eigen::VectorXd -> std::vector<double>, Eigen::Isometry3d -> Pose {xyz, wxyz};
//   * errors are std::runtime_error (PRINT_AND_THROW, trajopt_common/macros.h:90-98); solver failures are status codes;
//   * sco::ModelType is resolved BY NAME (the reference's name table is permuted against its enum, SURVEY.md section 8b).
// Header only; link with -ltrajopt_b200.  Everything lives in namespace trajopt_b200 so that a shim inside the
// reference tree can alias it (namespace tb = trajopt_b200).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <filesystem>
#include <fstream>
#include <functional>
#include <map>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "trajopt_b200.h"

namespace trajopt_b200 {

using DblVec = std::vector<double>;  // sco::DblVec, trajopt_sco/include/trajopt_sco/sco_common.hpp:17
using IntVec = std::vector<int>;

namespace sco {

// trajopt_sco/include/trajopt_sco/optimizers.hpp:25-33
enum OptStatus : int {
  OPT_CONVERGED = TB200_OPT_CONVERGED,
  OPT_SCO_ITERATION_LIMIT = TB200_OPT_SCO_ITERATION_LIMIT,
  OPT_PENALTY_ITERATION_LIMIT = TB200_OPT_PENALTY_ITERATION_LIMIT,
  OPT_TIME_LIMIT = TB200_OPT_TIME_LIMIT,
  OPT_FAILED = TB200_OPT_FAILED,
  INVALID = TB200_OPT_INVALID
};

// optimizers.hpp:92-135 (same names, same defaults)
struct BasicTrustRegionSQPParameters {
  double improve_ratio_threshold = 0.25;
  double min_trust_box_size = 1e-4;
  double min_approx_improve = 1e-4;
  double min_approx_improve_frac = std::numeric_limits<double>::lowest();
  int max_iter = 50;
  double trust_shrink_ratio = 0.1;
  double trust_expand_ratio = 1.5;
  double cnt_tolerance = 1e-4;
  double max_merit_coeff_increases = 5;
  int max_qp_solver_failures = 3;
  double merit_coeff_increase_ratio = 10;
  double initial_merit_error_coeff = 10;
  bool inflate_constraints_individually = true;
  double trust_box_size = 1e-1;
  double max_time = std::numeric_limits<double>::max();  // seconds (DESIGN.md section 6: one device clock per batch)
  // optimizers.hpp:127-129: write log_dir/<problem>/trajopt_{solver,vars,costs,constraints}.log (OptimizeWithParams from
  // pci.opt_info or with callbacks; one directory per problem of the batch).  Not read from JSON, as in the reference.
  bool log_results = false;
  std::string log_dir = "/tmp";
};

// optimizers.hpp:40-59
struct OptResults {
  DblVec x;  // [T*D], trajToDblVec order
  OptStatus status = INVALID;
  double total_cost = 0;
  DblVec cost_vals, cnt_viols;
  int n_func_evals = 0, n_qp_solves = 0;
};

// solver_interface.hpp:229-236.  Only the OSQP-equivalent device solver exists here.
enum class ModelType { GUROBI, OSQP, QPOASES, BPMPD, AUTO_SOLVER };
inline ModelType modelTypeFromName(const std::string& name) {
  if (name == "GUROBI") return ModelType::GUROBI;
  if (name == "OSQP") return ModelType::OSQP;
  if (name == "QPOASES") return ModelType::QPOASES;
  if (name == "BPMPD") return ModelType::BPMPD;
  if (name == "AUTO_SOLVER") return ModelType::AUTO_SOLVER;
  throw std::runtime_error("invalid solver name:\"" + name + "\"");  // solver_interface.cpp:243-258
}

}  // namespace sco

namespace trajopt {

// problem_description.hpp:34-41
enum TermType : int { TT_INVALID = 0, TT_COST = 0x1, TT_CNT = 0x2, TT_USE_TIME = 0x4 };

struct Pose {  // Eigen::Isometry3d stand-in
  double xyz[3] = {0, 0, 0};
  double wxyz[4] = {1, 0, 0, 0};
};

// What ConstructProblem takes from pci.kin / pci.env (problem_description.cpp:410-460, 553-592): the manipulator
// chain, its limits and the collision geometry of its links.
struct RobotModel {
  struct Joint {
    std::string child_link;  // name of the frame this joint creates
    int parent = -1;         // index of the parent joint/frame, -1 = scene root
    int type = TB200_JOINT_FIXED;
    int q_index = -1;        // column of the trajectory
    Pose origin;
    double axis[3] = {0, 0, 1};
  };
  struct Sphere {
    std::string link;
    double center[3] = {0, 0, 0};
    double radius = 0;
  };
  std::vector<Joint> joints;  // topologically ordered
  DblVec lower, upper;        // kin->getLimits()
  std::vector<Sphere> spheres;
  int numJoints() const { return static_cast<int>(lower.size()); }
  int linkIndex(const std::string& name) const {
    for (size_t i = 0; i < joints.size(); ++i)
      if (joints[i].child_link == name) return static_cast<int>(i);
    throw std::runtime_error("link \"" + name + "\" is not part of the manipulator model");
  }
};

// problem_description.hpp:123-157 (use_time / dt limits are not on the device path)
struct BasicInfo {
  int n_steps = -1;
  std::string manip;
  IntVec fixed_timesteps;
  IntVec fixed_dofs;
  sco::ModelType convex_solver = sco::ModelType::AUTO_SOLVER;
  bool use_time = false;
};

// problem_description.hpp:162-185.  data: JOINT_INTERPOLATED -> end states [B][D]; GIVEN_TRAJ -> [B][T][D];
// start: the current joint values of every problem [B][D] (pci.env->getCurrentJointValues in the reference).
struct InitInfo {
  enum Type : std::uint8_t { STATIONARY, JOINT_INTERPOLATED, GIVEN_TRAJ };
  Type type = STATIONARY;
  DblVec data;
  DblVec start;
};

struct ProblemConstructionInfo;
struct Flat;  // accumulates the POD description

// problem_description.hpp:199-230
struct TermInfo {
  using Ptr = std::shared_ptr<TermInfo>;
  std::string name;
  int term_type = TT_INVALID;
  virtual void hatch(Flat& flat, const ProblemConstructionInfo& pci) const = 0;
  virtual ~TermInfo() = default;
};

struct Flat {
  std::vector<tb200_term> terms;
  DblVec cart_targets;  // [B][n_slots][7]
  int n_slots = 0, batch = 0;
  int addTargets(const std::vector<Pose>& per_traj) {  // one static target per trajectory -> a slot
    if (static_cast<int>(per_traj.size()) != batch) throw std::runtime_error("cart_pose: one target pose per trajectory is required");
    DblVec grown(static_cast<size_t>(batch) * (n_slots + 1) * 7);
    for (int b = 0; b < batch; ++b) {
      for (int s = 0; s < n_slots; ++s)
        for (int k = 0; k < 7; ++k) grown[(static_cast<size_t>(b) * (n_slots + 1) + s) * 7 + k] = cart_targets[(static_cast<size_t>(b) * n_slots + s) * 7 + k];
      double* o = &grown[(static_cast<size_t>(b) * (n_slots + 1) + n_slots) * 7];
      for (int k = 0; k < 3; ++k) o[k] = per_traj[b].xyz[k];
      for (int k = 0; k < 4; ++k) o[3 + k] = per_traj[b].wxyz[k];
    }
    cart_targets.swap(grown);
    return n_slots++;
  }
};

namespace detail {
inline tb200_term blankTerm(int kind, int term_type, const std::string& name) {
  if (term_type != TT_COST && term_type != TT_CNT) throw std::runtime_error(name + ": term_type must be TT_COST or TT_CNT");
  tb200_term t{};
  t.kind = kind;
  t.role = (term_type == TT_COST) ? TB200_ROLE_COST : TB200_ROLE_CNT;
  return t;
}
inline void fill(double* dst, const DblVec& src, int n, double def, const std::string& what) {
  if (!src.empty() && static_cast<int>(src.size()) != n) throw std::runtime_error(what + " has the wrong size");
  for (int i = 0; i < n; ++i) dst[i] = src.empty() ? def : src[i];
}
}  // namespace detail

// JointPos/Vel/AccTermInfo, problem_description.hpp:430-560; hatch step clamping problem_description.cpp:1078-1106,
// 1197-1224, 1393-1421 (last_step <= -1: to the end; velocity needs two steps, acceleration three).
struct JointTermInfoBase : TermInfo {
  DblVec coeffs, targets, upper_tols, lower_tols;
  int first_step = 0, last_step = -1;
  int order_ = 0;
  void hatch(Flat& flat, const ProblemConstructionInfo& pci) const override;
};
struct JointPosTermInfo : JointTermInfoBase { JointPosTermInfo() { order_ = 0; name = "joint_pos"; } };
struct JointVelTermInfo : JointTermInfoBase { JointVelTermInfo() { order_ = 1; name = "joint_vel"; } };
struct JointAccTermInfo : JointTermInfoBase { JointAccTermInfo() { order_ = 2; name = "joint_acc"; } };

// CartPoseTermInfo, problem_description.hpp:330-376 (static target; tolerances / error_function not on the device path)
struct CartPoseTermInfo : TermInfo {
  int timestep = 0;
  double pos_coeffs[3] = {1, 1, 1}, rot_coeffs[3] = {1, 1, 1};
  std::string source_frame;
  Pose source_frame_offset;
  std::vector<Pose> target;  // target_frame * target_frame_offset in the scene root, one per trajectory
  CartPoseTermInfo() { name = "cart_pose"; }
  void hatch(Flat& flat, const ProblemConstructionInfo& pci) const override;
};

// CartVelTermInfo, problem_description.hpp:383-398
struct CartVelTermInfo : TermInfo {
  int first_step = -1, last_step = -1;
  std::string link;
  double max_displacement = 0;
  CartVelTermInfo() { name = "cart_vel"; }
  void hatch(Flat& flat, const ProblemConstructionInfo& pci) const override;
};

// AvoidSingularityTermInfo, problem_description.hpp:637-659 (without subset_kin_): one object per step on the smallest
// singular value of `link`'s geometric Jacobian; a TT_COST is an ABS cost, a TT_CNT an INEQ constraint.  hatch throws
// for more than one coefficient, an unknown link and steps outside the trajectory (the defaults -1 included).
struct AvoidSingularityTermInfo : TermInfo {
  std::string link;
  int first_step = -1, last_step = -1;
  DblVec coeffs;  // empty: no scaling; one element: the scale of err and gradient
  double lambda = 0.1;
  AvoidSingularityTermInfo() { name = "avoid_singularity"; }
  void hatch(Flat& flat, const ProblemConstructionInfo& pci) const override;
};

// CollisionTermInfo, problem_description.hpp:600-659 + trajopt_common TrajOptCollisionConfig (collision_types.h:120-170)
struct CollisionTermInfo : TermInfo {
  int first_step = 0, last_step = -1;
  IntVec fixed_steps;
  int evaluator_type = TB200_COLL_DISCRETE;  // CollisionEvaluatorType
  double collision_margin = 0.025;           // "dist_pen" / safety margin
  double collision_coeff = 20;
  double collision_margin_buffer = 0.01;
  double longest_valid_segment_length = 0.005;
  CollisionTermInfo() { name = "collision"; }
  void hatch(Flat& flat, const ProblemConstructionInfo& pci) const override;
};

// problem_description.hpp:235-259
struct ProblemConstructionInfo {
  BasicInfo basic_info;
  sco::BasicTrustRegionSQPParameters opt_info;
  std::vector<TermInfo::Ptr> cost_infos, cnt_infos;
  InitInfo init_info;
  std::shared_ptr<const RobotModel> kin;  // stands in for pci.kin + pci.env
  int batch = 1;
  DblVec obstacles;  // static world spheres (x, y, z, r): [B][O][4] or [O][4]
  int n_obstacles = 0;
  bool obstacles_per_problem = true;
  // Multi-start (not in the reference): batch = problems * seeds_per_problem; trajectories [p*G, (p+1)*G) are the seeds
  // of problem p (they normally differ only in init_info).  stop_seeds_on_converged: once a seed converges, its
  // siblings end at their next SQP iteration top (tb200_problem_desc.group_stop).  OptimizeProblemMultiStart.
  int seeds_per_problem = 1;
  bool stop_seeds_on_converged = false;
};

inline void JointTermInfoBase::hatch(Flat& flat, const ProblemConstructionInfo& pci) const {
  const int T = pci.basic_info.n_steps, D = pci.kin->numJoints();
  int first = first_step, last = last_step;
  if (last <= -1) last = T - 1;
  if ((T - 1 - order_) <= first) first = T - 1 - order_;
  if ((T - 1) <= last) last = T - 1;
  if (order_ > 0 && last == first) last += order_;
  if (last < first) std::swap(first, last);
  tb200_term t = detail::blankTerm(TB200_TERM_JOINT_POS + order_, term_type, name);
  t.first_step = first;
  t.last_step = last;
  detail::fill(t.coeffs, coeffs, D, 1.0, name + ": coeffs");
  detail::fill(t.targets, targets, D, 0.0, name + ": targets");
  detail::fill(t.upper_tols, upper_tols, D, 0.0, name + ": upper_tols");
  detail::fill(t.lower_tols, lower_tols, D, 0.0, name + ": lower_tols");
  flat.terms.push_back(t);
}
inline void CartPoseTermInfo::hatch(Flat& flat, const ProblemConstructionInfo& pci) const {
  tb200_term t = detail::blankTerm(TB200_TERM_CART_POSE, term_type, name);
  t.first_step = t.last_step = timestep;
  t.link = pci.kin->linkIndex(source_frame);
  for (int k = 0; k < 3; ++k) {
    t.source_offset[k] = source_frame_offset.xyz[k];
    t.pos_coeffs[k] = pos_coeffs[k];
    t.rot_coeffs[k] = rot_coeffs[k];
  }
  for (int k = 0; k < 4; ++k) t.source_offset[3 + k] = source_frame_offset.wxyz[k];
  t.target_pose[3] = 1.0;  // unused: the target is read from the per-trajectory slot
  t.target_slot = flat.addTargets(target);
  flat.terms.push_back(t);
}
inline void AvoidSingularityTermInfo::hatch(Flat& flat, const ProblemConstructionInfo& pci) const {
  tb200_term t = detail::blankTerm(TB200_TERM_AVOID_SINGULARITY, term_type, name);
  const int T = pci.basic_info.n_steps;
  if (coeffs.size() > 1) throw std::runtime_error(name + ": coeffs has more than one element");
  if (first_step < 0 || last_step >= T || first_step > last_step)
    throw std::runtime_error(name + ": steps outside the trajectory");
  t.first_step = first_step;
  t.last_step = last_step;
  t.link = pci.kin->linkIndex(link);
  t.target_slot = -1;
  t.coeffs[0] = coeffs.empty() ? 1.0 : coeffs[0];
  t.lambda = lambda;
  flat.terms.push_back(t);
}
inline void CartVelTermInfo::hatch(Flat& flat, const ProblemConstructionInfo& pci) const {
  tb200_term t = detail::blankTerm(TB200_TERM_CART_VEL, term_type, name);
  const int T = pci.basic_info.n_steps;
  t.first_step = first_step < 0 ? 0 : first_step;
  t.last_step = (last_step < 0 || last_step > T - 2) ? T - 2 : last_step;  // pair t = (t, t+1)
  t.link = pci.kin->linkIndex(link);
  t.target_slot = -1;
  t.max_displacement = max_displacement;
  flat.terms.push_back(t);
}
inline void CollisionTermInfo::hatch(Flat& flat, const ProblemConstructionInfo& pci) const {
  tb200_term t = detail::blankTerm(TB200_TERM_COLLISION, term_type, name);
  const int T = pci.basic_info.n_steps;
  t.first_step = first_step;
  t.last_step = (last_step <= -1 || last_step > T - 1) ? T - 1 : last_step;
  t.evaluator_type = evaluator_type;
  if (fixed_steps.size() > 8) throw std::runtime_error(name + ": more than 8 fixed_steps");
  t.n_fixed_steps = static_cast<int>(fixed_steps.size());
  for (size_t i = 0; i < fixed_steps.size(); ++i) t.fixed_steps[i] = fixed_steps[i];
  t.margin = collision_margin;
  t.coeff = collision_coeff;
  t.margin_buffer = collision_margin_buffer;
  t.longest_valid_segment_length = longest_valid_segment_length;
  flat.terms.push_back(t);
}

// The flattened description with everything it points to (kept alive together).
struct FlatProblem {
  tb200_problem_desc desc{};
  std::vector<tb200_segment> segments;
  std::vector<tb200_sphere> spheres;
  DblVec lower, upper, init_traj, cart_targets, obstacles;
  std::vector<tb200_term> terms;
  std::vector<int32_t> fixed_timesteps, fixed_dofs;
  int n_costs_terms = 0;
  std::vector<std::string> term_names;  // TermInfo::name of every term, in terms order
  bool log_results = false;             // pci.opt_info.log_results / log_dir
  std::string log_dir;
  std::shared_ptr<const RobotModel> kin;  // pci.kin (WriteCallback's FK)
};

// The C ABI's form of one set of optimizer parameters (log_results / log_dir stay on the host).
inline tb200_sqp_params ToSqpParams(const sco::BasicTrustRegionSQPParameters& p) {
  tb200_sqp_params s{};
  s.improve_ratio_threshold = p.improve_ratio_threshold;
  s.min_trust_box_size = p.min_trust_box_size;
  s.min_approx_improve = p.min_approx_improve;
  s.min_approx_improve_frac = p.min_approx_improve_frac;
  s.max_iter = p.max_iter;
  s.max_qp_solver_failures = p.max_qp_solver_failures;
  s.trust_shrink_ratio = p.trust_shrink_ratio;
  s.trust_expand_ratio = p.trust_expand_ratio;
  s.cnt_tolerance = p.cnt_tolerance;
  s.max_merit_coeff_increases = p.max_merit_coeff_increases;
  s.merit_coeff_increase_ratio = p.merit_coeff_increase_ratio;
  s.initial_merit_error_coeff = p.initial_merit_error_coeff;
  s.trust_box_size = p.trust_box_size;
  s.inflate_constraints_individually = p.inflate_constraints_individually ? 1 : 0;
  s.reserved = 0;
  s.max_time = p.max_time;
  return s;
}
// The per-trajectory table (tb200_problem_set_sqp_params_per_traj) of a batch of `batch` problems, row b from params[b];
// throws std::invalid_argument unless there is exactly one entry per problem.
inline std::vector<tb200_sqp_params> SqpParamRows(int batch, const std::vector<sco::BasicTrustRegionSQPParameters>& params) {
  if (params.size() != static_cast<size_t>(batch))
    throw std::invalid_argument("per-problem optimizer parameters: " + std::to_string(params.size()) +
                                " entries for a batch of " + std::to_string(batch));
  std::vector<tb200_sqp_params> rows;
  rows.reserve(params.size());
  for (const sco::BasicTrustRegionSQPParameters& p : params) rows.push_back(ToSqpParams(p));
  return rows;
}

// The part of ConstructProblem (problem_description.cpp:410-542) that does not need the device: checks, initial
// trajectory (InitInfo, :330-408), term hatching into the POD description (cost_infos first, then cnt_infos).
inline std::shared_ptr<FlatProblem> FlattenProblem(const ProblemConstructionInfo& pci) {
  if (!pci.kin) throw std::runtime_error("ProblemConstructionInfo: no kinematics");
  const RobotModel& kin = *pci.kin;
  const int T = pci.basic_info.n_steps, D = kin.numJoints(), B = pci.batch;
  if (T < 1) throw std::runtime_error("basic_info.n_steps must be positive");
  if (pci.basic_info.use_time) throw std::runtime_error("use_time problems are not on the device path");
  if (pci.basic_info.convex_solver != sco::ModelType::OSQP && pci.basic_info.convex_solver != sco::ModelType::AUTO_SOLVER)
    throw std::runtime_error("the device path implements the OSQP-equivalent solver only");
  auto fp = std::make_shared<FlatProblem>();
  for (const RobotModel::Joint& j : kin.joints) {
    tb200_segment s{};
    s.parent = j.parent;
    s.joint_type = j.type;
    s.q_index = j.q_index;
    for (int k = 0; k < 3; ++k) { s.origin_xyz[k] = j.origin.xyz[k]; s.axis[k] = j.axis[k]; }
    for (int k = 0; k < 4; ++k) s.origin_wxyz[k] = j.origin.wxyz[k];
    fp->segments.push_back(s);
  }
  for (const RobotModel::Sphere& sp : kin.spheres) {
    tb200_sphere s{};
    s.segment = kin.linkIndex(sp.link);
    for (int k = 0; k < 3; ++k) s.center[k] = sp.center[k];
    s.radius = sp.radius;
    fp->spheres.push_back(s);
  }
  fp->lower = kin.lower;
  fp->upper = kin.upper;
  // ---- InitInfo (problem_description.cpp:330-408)
  const InitInfo& ii = pci.init_info;
  fp->init_traj.assign(static_cast<size_t>(B) * T * D, 0.0);
  if (ii.type == InitInfo::GIVEN_TRAJ) {
    if (ii.data.size() != fp->init_traj.size()) throw std::runtime_error("Initial trajectory has the wrong size");
    fp->init_traj = ii.data;
  } else {
    if (ii.start.size() != static_cast<size_t>(B) * D) throw std::runtime_error("InitInfo.start: one joint state per problem is required");
    if (ii.type == InitInfo::JOINT_INTERPOLATED && ii.data.size() != static_cast<size_t>(B) * D)
      throw std::runtime_error("init_info.data has the wrong size for JOINT_INTERPOLATED");
    for (int b = 0; b < B; ++b)
      for (int t = 0; t < T; ++t)
        for (int d = 0; d < D; ++d) {
          const double s = ii.start[static_cast<size_t>(b) * D + d];
          double v = s;
          if (ii.type == InitInfo::JOINT_INTERPOLATED && T > 1) {  // LinSpaced per joint, :351-355
            const double e = ii.data[static_cast<size_t>(b) * D + d];
            v = (t == T - 1) ? e : s + t * ((e - s) / (T - 1));
          }
          fp->init_traj[(static_cast<size_t>(b) * T + t) * D + d] = v;
        }
  }
  // ---- terms: cost_infos first, then cnt_infos (problem_description.cpp:462-484)
  Flat flat;
  flat.batch = B;
  for (const auto& ti : pci.cost_infos) {
    if (ti->term_type != TT_COST) throw std::runtime_error(ti->name + ": a cost_info must have term_type TT_COST");
    ti->hatch(flat, pci);
  }
  fp->n_costs_terms = static_cast<int>(flat.terms.size());
  for (const auto& ti : pci.cnt_infos) {
    if (ti->term_type != TT_CNT) throw std::runtime_error(ti->name + ": a cnt_info must have term_type TT_CNT");
    ti->hatch(flat, pci);
  }
  for (const auto* infos : {&pci.cost_infos, &pci.cnt_infos})
    for (const auto& ti : *infos) fp->term_names.push_back(ti->name);  // (every hatch adds one term)
  fp->log_results = pci.opt_info.log_results;
  fp->kin = pci.kin;
  fp->log_dir = pci.opt_info.log_dir;
  fp->terms = flat.terms;
  fp->cart_targets = flat.cart_targets;
  {
    const size_t want = static_cast<size_t>(pci.obstacles_per_problem ? B : 1) * static_cast<size_t>(pci.n_obstacles) * 4;
    if (pci.obstacles.size() != want)
      throw std::runtime_error("obstacles has " + std::to_string(pci.obstacles.size()) + " values, expected " + std::to_string(want) +
                               " ([B or 1][n_obstacles][4])");
  }
  fp->obstacles = pci.obstacles;
  fp->fixed_timesteps.assign(pci.basic_info.fixed_timesteps.begin(), pci.basic_info.fixed_timesteps.end());
  fp->fixed_dofs.assign(pci.basic_info.fixed_dofs.begin(), pci.basic_info.fixed_dofs.end());
  tb200_problem_desc& d = fp->desc;
  d.robot.n_dof = D;
  d.robot.n_segments = static_cast<int32_t>(fp->segments.size());
  d.robot.segments = fp->segments.data();
  d.robot.lower = fp->lower.data();
  d.robot.upper = fp->upper.data();
  d.robot.n_spheres = static_cast<int32_t>(fp->spheres.size());
  d.robot.spheres = fp->spheres.data();
  d.n_steps = T;
  d.batch = B;
  d.n_terms = static_cast<int32_t>(fp->terms.size());
  d.terms = fp->terms.data();
  d.n_fixed_timesteps = static_cast<int32_t>(fp->fixed_timesteps.size());
  d.fixed_timesteps = fp->fixed_timesteps.data();
  d.n_fixed_dofs = static_cast<int32_t>(fp->fixed_dofs.size());
  d.fixed_dofs = fp->fixed_dofs.data();
  d.n_cart_targets = flat.n_slots;
  d.init_traj = fp->init_traj.data();
  d.cart_targets = fp->cart_targets.empty() ? nullptr : fp->cart_targets.data();
  d.n_obstacles = pci.n_obstacles;
  d.obstacles_per_traj = pci.obstacles_per_problem ? 1 : 0;
  d.obstacles = fp->obstacles.empty() ? nullptr : fp->obstacles.data();
  tb200_default_qp_settings(&d.qp);  // OSQPModelConfig::setDefaultOSQPSettings, osqp_interface.cpp:78-90
  d.sqp = ToSqpParams(pci.opt_info);
  d.group_size = pci.seeds_per_problem;
  d.group_stop = pci.stop_seeds_on_converged ? 1 : 0;
  return fp;
}

// The batched TrajOptProb: owns the device handle (problem_description.hpp:68-107 for one problem).
class TrajOptProb {
public:
  using Ptr = std::shared_ptr<TrajOptProb>;
  TrajOptProb(std::shared_ptr<FlatProblem> flat, int device) : flat_(std::move(flat)) {
    if (tb200_problem_create(&flat_->desc, device, &handle_) != TB200_OK) throw std::runtime_error(tb200_last_error());
    if (tb200_problem_layout(handle_, &layout_) != TB200_OK) throw std::runtime_error(tb200_last_error());
  }
  ~TrajOptProb() { tb200_problem_destroy(handle_); }
  TrajOptProb(const TrajOptProb&) = delete;
  TrajOptProb& operator=(const TrajOptProb&) = delete;
  int GetNumSteps() const { return flat_->desc.n_steps; }
  int GetNumDOF() const { return flat_->desc.robot.n_dof; }
  int GetBatch() const { return flat_->desc.batch; }
  int GetSeedsPerProblem() const { return flat_->desc.group_size > 1 ? flat_->desc.group_size : 1; }
  const DblVec& GetInitTraj() const { return flat_->init_traj; }
  const tb200_sqp_params& sqpParams() const { return flat_->desc.sqp; }  // = pci.opt_info
  int getNumCosts() const { return layout_.n_costs; }
  int getNumConstraints() const { return layout_.n_cnts; }
  tb200_problem* handle() const { return handle_; }
  const FlatProblem& flat() const { return *flat_; }

private:
  std::shared_ptr<FlatProblem> flat_;
  tb200_problem* handle_ = nullptr;
  tb200_layout layout_{};
};

// trajopt::ConstructProblem(pci), problem_description.hpp:661 / problem_description.cpp:410-542
inline TrajOptProb::Ptr ConstructProblem(const ProblemConstructionInfo& pci, int device = 0) {
  return std::make_shared<TrajOptProb>(FlattenProblem(pci), device);
}

// BasicTrustRegionSQP::optimize() for every problem of the batch (optimizers.cpp:699-991) with the given parameters: what
// `sco::BasicTrustRegionSQP opt(prob); opt.getParameters() = params; opt.initialize(...); opt.optimize(); opt.results()`
// returns, per problem.
namespace detail {
// Sets the optimizer parameters of the next solve: one row for every problem, or one row per problem (B > 1).
inline void setSqpParams(TrajOptProb& prob, const std::vector<tb200_sqp_params>& rows) {
  const int rc = rows.size() == 1 ? tb200_problem_set_sqp_params(prob.handle(), rows.data())
                                  : tb200_problem_set_sqp_params_per_traj(prob.handle(), rows.data());
  if (rc != TB200_OK) throw std::runtime_error(tb200_last_error());
}
inline std::vector<sco::OptResults> solveBatch(TrajOptProb& prob);
}  // namespace detail
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob, const tb200_sqp_params& params) {
  detail::setSqpParams(prob, {params});
  return detail::solveBatch(prob);
}
inline std::vector<sco::OptResults> detail::solveBatch(TrajOptProb& prob) {
  const size_t B = prob.GetBatch(), N = static_cast<size_t>(prob.GetNumSteps()) * prob.GetNumDOF();
  const size_t nc = prob.getNumCosts(), nk = prob.getNumConstraints();
  DblVec x(B * N), total(B), cv(B * (nc ? nc : 1)), kv(B * (nk ? nk : 1));
  std::vector<int32_t> status(B), nqp(B), nfe(B);
  tb200_results r{};
  r.x = x.data(); r.status = status.data(); r.total_cost = total.data();
  r.cost_vals = nc ? cv.data() : nullptr; r.cnt_viols = nk ? kv.data() : nullptr;
  r.n_qp_solves = nqp.data(); r.n_func_evals = nfe.data();
  if (tb200_solve_batch(prob.handle(), &r) != TB200_OK) throw std::runtime_error(tb200_last_error());
  std::vector<sco::OptResults> out(B);
  for (size_t b = 0; b < B; ++b) {
    out[b].x.assign(x.begin() + b * N, x.begin() + (b + 1) * N);
    out[b].status = static_cast<sco::OptStatus>(status[b]);
    out[b].total_cost = total[b];
    out[b].cost_vals.assign(cv.begin() + b * nc, cv.begin() + (b + 1) * nc);
    out[b].cnt_viols.assign(kv.begin() + b * nk, kv.begin() + (b + 1) * nk);
    out[b].n_qp_solves = nqp[b];
    out[b].n_func_evals = nfe[b];
  }
  return out;
}
// ... with the problem description's own parameters (pci.opt_info; with its log_results, log_dir/<problem>/trajopt_*.log
// are written as by the overload with callbacks)
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob);

// trajopt::OptimizeProblem(prob) (problem_description.hpp:665, problem_description.cpp:392-408).  The reference's function
// does NOT run with pci.opt_info: it builds a fresh BasicTrustRegionSQP and overrides four parameters (max_iter 40,
// min_approx_improve_frac 1e-3, improve_ratio_threshold 0.2, initial_merit_error_coeff 20) on top of the optimizer's
// DEFAULTS.  Reproduced here, so that the same description gives the same iterates; OptimizeWithParams is the entry point
// that honours pci.opt_info.
inline std::vector<sco::OptResults> OptimizeProblem(TrajOptProb& prob) {
  tb200_sqp_params p;
  tb200_default_sqp_params(&p);
  p.max_iter = 40;
  p.min_approx_improve_frac = .001;
  p.improve_ratio_threshold = .2;
  p.initial_merit_error_coeff = 20;
  return OptimizeWithParams(prob, p);
}

// ---- SQP iteration log, optimizer callbacks and log_results (DESIGN.md section 4.7) ----------------------------------

// The log of the last solve (tb200_fetch_sqp_log) on the host: R records per problem, [B][R](...) like the C struct.
struct SqpLog {
  int B = 0, R = 0, n_costs = 0, n_cnts = 0, N = 0;
  bool with_x = false;
  std::vector<int32_t> n_records, n_dropped, kind, merit_round, iter, qp_status, admm_iters, polish, action, ended;
  DblVec trust_box_size, old_merit, model_merit, new_merit, merit_coeffs, model_cost_vals, model_cnt_viols, old_cost_vals,
      old_cnt_viols, new_cost_vals, new_cnt_viols, new_x;
  size_t at(size_t b, size_t r) const { return b * R + r; }
};

inline SqpLog FetchSqpLog(TrajOptProb& prob, int capacity, bool with_x) {
  SqpLog L;
  L.B = prob.GetBatch(); L.R = capacity; L.n_costs = prob.getNumCosts(); L.n_cnts = prob.getNumConstraints();
  L.N = prob.GetNumSteps() * prob.GetNumDOF(); L.with_x = with_x;
  const size_t BR = static_cast<size_t>(L.B) * L.R;
  for (auto* v : {&L.kind, &L.merit_round, &L.iter, &L.qp_status, &L.admm_iters, &L.polish, &L.action, &L.ended}) v->resize(BR);
  for (auto* v : {&L.trust_box_size, &L.old_merit, &L.model_merit, &L.new_merit}) v->resize(BR);
  L.n_records.resize(L.B); L.n_dropped.resize(L.B);
  L.merit_coeffs.resize(BR * L.n_cnts); L.model_cnt_viols.resize(BR * L.n_cnts); L.old_cnt_viols.resize(BR * L.n_cnts);
  L.new_cnt_viols.resize(BR * L.n_cnts);
  L.model_cost_vals.resize(BR * L.n_costs); L.old_cost_vals.resize(BR * L.n_costs); L.new_cost_vals.resize(BR * L.n_costs);
  if (with_x) L.new_x.resize(BR * L.N);
  auto p = [](DblVec& v) { return v.empty() ? nullptr : v.data(); };
  tb200_sqp_log o{};
  o.n_records = L.n_records.data(); o.n_dropped = L.n_dropped.data(); o.kind = L.kind.data();
  o.merit_round = L.merit_round.data(); o.iter = L.iter.data(); o.trust_box_size = p(L.trust_box_size);
  o.qp_status = L.qp_status.data(); o.admm_iters = L.admm_iters.data(); o.polish = L.polish.data();
  o.action = L.action.data(); o.ended = L.ended.data();
  o.old_merit = p(L.old_merit); o.model_merit = p(L.model_merit); o.new_merit = p(L.new_merit);
  o.merit_coeffs = p(L.merit_coeffs); o.model_cost_vals = p(L.model_cost_vals); o.model_cnt_viols = p(L.model_cnt_viols);
  o.old_cost_vals = p(L.old_cost_vals); o.old_cnt_viols = p(L.old_cnt_viols);
  o.new_cost_vals = p(L.new_cost_vals); o.new_cnt_viols = p(L.new_cnt_viols); o.new_x = p(L.new_x);
  if (tb200_fetch_sqp_log(prob.handle(), &o) != TB200_OK) throw std::runtime_error(tb200_last_error());
  return L;
}

// sco::Optimizer::Callback (optimizers.hpp:83) for a batch: the problem index says whose state the results are.
using Callback = std::function<void(TrajOptProb*, std::size_t problem, sco::OptResults&)>;

// Calls the callbacks as the reference's optimizer does for problem b (optimizers.cpp:754, 978): once at the top of every
// SQP iteration that ran a QP - a new (merit_round, iter) in the log - and once at the end with final.  At a top the
// results hold what the reference's hold there: the last accepted point and its exact values, and the QP solves and
// function evaluations so far (a failed QP evaluates nothing); at the first top, before the first evaluation, the value
// vectors are empty and the counts 0.  The log must hold the points (with_x).  A truncated log throws, naming the
// problem, unless allow_truncated (then the replay stops with the records kept).
inline void ReplayCallbacks(TrajOptProb* prob, const SqpLog& L, std::size_t b, sco::OptResults final_results,
                            const std::vector<Callback>& callbacks, bool allow_truncated = false) {
  if (L.n_dropped[b] > 0 && !allow_truncated)
    throw std::runtime_error("SQP log of problem " + std::to_string(b) + " is truncated: " + std::to_string(L.n_dropped[b]) +
                             " records did not fit a capacity of " + std::to_string(L.R));
  if (!L.with_x) throw std::runtime_error("replaying callbacks needs a log recorded with x");
  const size_t N = L.N, nc = L.n_costs, nk = L.n_cnts;
  sco::OptResults cur;
  cur.status = sco::INVALID;
  int last_round = -1, last_iter = -1, n_qp = 0, n_fe = 0;
  for (int r = 0; r < L.n_records[b]; ++r) {
    const size_t i = L.at(b, r);
    if (L.kind[i] == 0) {  // the state after the first evaluation: the first top sees its point, no values yet
      cur.x.assign(L.new_x.begin() + i * N, L.new_x.begin() + (i + 1) * N);
      continue;
    }
    if (L.merit_round[i] != last_round || L.iter[i] != last_iter) {
      last_round = L.merit_round[i];
      last_iter = L.iter[i];
      cur.n_qp_solves = n_qp;
      cur.n_func_evals = n_fe;
      for (const Callback& cb : callbacks) {
        sco::OptResults view = cur;
        cb(prob, b, view);
      }
    }
    if (n_fe == 0) {  // the first iteration evaluates the start point (optimizers.cpp:761-767)
      const size_t i0 = L.at(b, 0);
      cur.cost_vals.assign(L.new_cost_vals.begin() + i0 * nc, L.new_cost_vals.begin() + (i0 + 1) * nc);
      cur.cnt_viols.assign(L.new_cnt_viols.begin() + i0 * nk, L.new_cnt_viols.begin() + (i0 + 1) * nk);
      n_fe = 1;
    }
    ++n_qp;
    if (L.action[i] != 3) ++n_fe;
    if (L.action[i] == 1) {
      cur.x.assign(L.new_x.begin() + i * N, L.new_x.begin() + (i + 1) * N);
      cur.cost_vals.assign(L.new_cost_vals.begin() + i * nc, L.new_cost_vals.begin() + (i + 1) * nc);
      cur.cnt_viols.assign(L.new_cnt_viols.begin() + i * nk, L.new_cnt_viols.begin() + (i + 1) * nk);
    }
  }
  for (const Callback& cb : callbacks) {
    sco::OptResults view = final_results;
    cb(prob, b, view);
  }
}

// Names the reference gives the variables (problem_description.cpp:573-578) and the objects (TermInfo::hatch: the term's
// name; collision objects "<name>_<step>", :1758-1832).
inline std::vector<std::string> VarNames(int T, int D) {
  std::vector<std::string> v;
  for (int t = 0; t < T; ++t)
    for (int d = 0; d < D; ++d) v.push_back("j_" + std::to_string(t) + "_" + std::to_string(d));
  return v;
}
inline void ObjectNames(const TrajOptProb& prob, std::vector<std::string>& cost_names, std::vector<std::string>& cnt_names) {
  const int nc = prob.getNumCosts(), nk = prob.getNumConstraints();
  std::vector<int32_t> term(nc + nk + 1), step(nc + nk + 1);
  if (tb200_problem_objects(prob.handle(), term.data(), step.data()) != TB200_OK) throw std::runtime_error(tb200_last_error());
  const FlatProblem& f = prob.flat();
  cost_names.clear();
  cnt_names.clear();
  for (int i = 0; i < nc + nk; ++i) {
    const tb200_term& t = f.terms[term[i]];
    std::string n = f.term_names[term[i]];
    if (t.kind == TB200_TERM_COLLISION) n += "_" + std::to_string(step[i]);
    if (t.kind == TB200_TERM_CART_VEL && t.role == TB200_ROLE_CNT) n = "CartVel";  // :1044-1052 names its constraints so
    (i < nc ? cost_names : cnt_names).push_back(n);
  }
}

// log_results for problem b: dir/trajopt_{solver,vars,costs,constraints}.log, one line per successful QP with the header
// before the first, in the reference's formats (BasicTrustRegionSQPResults::write*, optimizers.cpp:533-647).
inline void WriteLogResults(const SqpLog& L, std::size_t b, const std::string& dir, const std::vector<std::string>& var_names,
                            const std::vector<std::string>& cost_names, const std::vector<std::string>& cnt_names) {
  std::filesystem::create_directories(dir);
  const char* files[4] = {"/trajopt_solver.log", "/trajopt_vars.log", "/trajopt_costs.log", "/trajopt_constraints.log"};
  std::FILE* f[4];
  for (int k = 0; k < 4; ++k)
    if (!(f[k] = std::fopen((dir + files[k]).c_str(), "w"))) throw std::runtime_error("cannot open " + dir + files[k]);
  const size_t N = L.N, nc = L.n_costs, nk = L.n_cnts;
  bool header = true;
  for (int r = 0; r < L.n_records[b]; ++r) {
    const size_t i = L.at(b, r);
    if (L.kind[i] != 1 || L.action[i] == 3) continue;  // the reference logs successful QPs only
    const double old_m = L.old_merit[i], model_m = L.model_merit[i], new_m = L.new_merit[i];
    const double approx = old_m - model_m, exact = old_m - new_m;
    if (header) std::fprintf(f[0], "%s,%s,%s,%s,%s,%s\n", "DESCRIPTION", "oldexact", "new_exact", "dapprox", "dexact", "ratio");
    std::fprintf(f[0], "%s,%10.3e,%10.3e,%10.3e,%10.3e,%10.3e\n", "Solver", old_m, new_m, approx, exact, exact / approx);
    if (header) {
      std::fprintf(f[1], "%s", "NAMES");
      for (const auto& v : var_names) std::fprintf(f[1], ",%s", v.c_str());
      std::fprintf(f[1], "\n");
    }
    std::fprintf(f[1], "%s", "VALUES");
    for (size_t k = 0; k < N && L.with_x; ++k) std::fprintf(f[1], ",%e", L.new_x[i * N + k]);
    std::fprintf(f[1], "\n");
    // costs (scale 1) and constraints (scaled by their merit coefficients)
    for (int c = 0; c < 2; ++c) {
      std::FILE* s = f[2 + c];
      const std::vector<std::string>& names = c ? cnt_names : cost_names;
      const size_t n = c ? nk : nc;
      const double* o = (c ? L.old_cnt_viols.data() : L.old_cost_vals.data()) + i * n;
      const double* m = (c ? L.model_cnt_viols.data() : L.model_cost_vals.data()) + i * n;
      const double* w = (c ? L.new_cnt_viols.data() : L.new_cost_vals.data()) + i * n;
      if (header) {
        std::fprintf(s, "%s", c ? "CONSTRAINT NAMES" : "COST NAMES");
        for (const auto& nm : names) std::fprintf(s, ",%s,%s,%s,%s", nm.c_str(), nm.c_str(), nm.c_str(), nm.c_str());
        std::fprintf(s, "\n");
        std::fprintf(s, "%s", "DESCRIPTION");
        for (size_t k = 0; k < names.size(); ++k) std::fprintf(s, ",%s,%s,%s,%s", "oldexact", "dapprox", "dexact", "ratio");
        std::fprintf(s, "\n");
      }
      std::fprintf(s, "%s", c ? "CONSTRAINTS" : "COSTS");
      for (size_t k = 0; k < n; ++k) {
        const double a = o[k] - m[k], e = o[k] - w[k], mu = c ? L.merit_coeffs[i * nk + k] : 1.0;
        const double ov = c ? mu * o[k] : o[k], av = c ? mu * a : a, ev = c ? mu * e : e;
        if (std::fabs(a) > 1e-8) std::fprintf(s, ",%e,%e,%e,%e", ov, av, ev, e / a);
        else std::fprintf(s, ",%e,%e,%e,%s", ov, av, ev, "nan");
      }
      std::fprintf(s, "\n");
    }
    header = false;
  }
  for (std::FILE* s : f) std::fclose(s);
}

// OptimizeWithParams with callbacks: the batch is solved with the SQP log on (with the points), then, per problem in
// batch order, the callbacks are replayed (ReplayCallbacks) and, with pci.opt_info's log_results,
// log_dir/<problem>/trajopt_*.log written.  The results are those of the solve without the log, bit for bit.
// log_capacity: records per problem; 0 sizes it from the parameters, 1 + max_iter x max_merit_coeff_increases (one QP per
// SQP iteration).  The device holds batch x capacity x (16 + 2 n_costs + 3 n_cnts + T*D) doubles while the log is on,
// and the host a copy of it: at configs[2] (batch 1024, 30 x 7 variables, 16 objects) 2560 bytes a record, 0.66 GB for
// the default 251 records.  When a problem needed more, the batch is solved once more with exactly the capacity the log
// counted (the solve is deterministic), unless allow_truncated asks for the prefix.
// With per-problem parameters the default capacity is the largest of those products, and log_results / log_dir are read
// per problem.
namespace detail {
// rows: one for every problem or one per problem (setSqpParams); log_dirs: per problem, the directory its log_results
// files go to ("": none), or empty for no files at all
inline std::vector<sco::OptResults> optimizeLogged(TrajOptProb& prob, const std::vector<tb200_sqp_params>& rows,
                                                   const std::vector<Callback>& callbacks,
                                                   const std::vector<std::string>& log_dirs, int log_capacity,
                                                   bool allow_truncated);
// log_dir/<problem> for every problem when log_results, else none
inline std::vector<std::string> logDirs(const TrajOptProb& prob, bool log_results, const std::string& log_dir) {
  std::vector<std::string> dirs;
  if (log_results)
    for (int b = 0; b < prob.GetBatch(); ++b) dirs.push_back(log_dir + "/" + std::to_string(b));
  return dirs;
}
inline std::vector<std::string> logDirs(const std::vector<sco::BasicTrustRegionSQPParameters>& params) {
  std::vector<std::string> dirs;
  bool any = false;
  for (size_t b = 0; b < params.size(); ++b) {
    dirs.push_back(params[b].log_results ? params[b].log_dir + "/" + std::to_string(b) : std::string());
    any = any || params[b].log_results;
  }
  return any ? dirs : std::vector<std::string>();
}
}  // namespace detail
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob, const tb200_sqp_params& params,
                                                       const std::vector<Callback>& callbacks, int log_capacity = 0,
                                                       bool allow_truncated = false) {
  return detail::optimizeLogged(prob, {params}, callbacks, detail::logDirs(prob, prob.flat().log_results, prob.flat().log_dir),
                                log_capacity, allow_truncated);
}
inline std::vector<sco::OptResults> detail::optimizeLogged(TrajOptProb& prob, const std::vector<tb200_sqp_params>& rows,
                                                           const std::vector<Callback>& callbacks,
                                                           const std::vector<std::string>& log_dirs, int log_capacity,
                                                           bool allow_truncated) {
  int cap = log_capacity;
  if (cap <= 0)
    for (const tb200_sqp_params& p : rows)
      cap = std::max(cap, 1 + std::max(p.max_iter, 1) * static_cast<int>(std::ceil(std::max(p.max_merit_coeff_increases, 1.0))));
  std::vector<sco::OptResults> out;
  SqpLog L;
  try {
    for (;;) {
      if (tb200_problem_set_sqp_log(prob.handle(), cap, 1) != TB200_OK) throw std::runtime_error(tb200_last_error());
      setSqpParams(prob, rows);
      out = solveBatch(prob);
      L = FetchSqpLog(prob, cap, true);
      int need = 0;
      for (int b = 0; b < L.B; ++b) need = std::max(need, L.n_records[b] + L.n_dropped[b]);
      if (need <= cap || allow_truncated) break;
      cap = need;
    }
  } catch (...) {
    tb200_problem_set_sqp_log(prob.handle(), 0, 0);
    throw;
  }
  tb200_problem_set_sqp_log(prob.handle(), 0, 0);
  std::vector<std::string> var_names, cost_names, cnt_names;
  if (!log_dirs.empty()) {
    var_names = VarNames(prob.GetNumSteps(), prob.GetNumDOF());
    ObjectNames(prob, cost_names, cnt_names);
  }
  for (size_t b = 0; b < out.size(); ++b) {
    ReplayCallbacks(&prob, L, b, out[b], callbacks, allow_truncated);
    if (!log_dirs.empty() && !log_dirs[b].empty()) WriteLogResults(L, b, log_dirs[b], var_names, cost_names, cnt_names);
  }
  return out;
}
// ... with the problem description's own parameters (pci.opt_info, its log_results and log_dir included)
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob, const std::vector<Callback>& callbacks) {
  return OptimizeWithParams(prob, prob.sqpParams(), callbacks);
}
// trajopt::OptimizeProblem with callbacks attached (problem_description.cpp:396-404 attaches its PlotCallback the same way);
// its fresh parameters keep the default log_results = false, as the reference's do
inline std::vector<sco::OptResults> OptimizeProblem(TrajOptProb& prob, const std::vector<Callback>& callbacks) {
  tb200_sqp_params p;
  tb200_default_sqp_params(&p);
  p.max_iter = 40;
  p.min_approx_improve_frac = .001;
  p.improve_ratio_threshold = .2;
  p.initial_merit_error_coeff = 20;
  return detail::optimizeLogged(prob, {p}, callbacks, {}, 0, false);
}
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob) {
  if (prob.flat().log_results)
    return detail::optimizeLogged(prob, {prob.sqpParams()}, {}, detail::logDirs(prob, true, prob.flat().log_dir), 0, false);
  return OptimizeWithParams(prob, prob.sqpParams());
}

// Per-problem parameters (not in the reference; DESIGN.md section 4.1): problem b of the batch runs under params[b], with
// exactly the results a batch solved under params[b] alone would give it.  One entry per problem of the batch, else
// std::invalid_argument.  With callbacks, or when some entry has log_results, the batch is solved with the SQP log as in
// the overload with callbacks; problem b's files go to params[b].log_dir/<b>.
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob,
                                                       const std::vector<sco::BasicTrustRegionSQPParameters>& params,
                                                       const std::vector<Callback>& callbacks, int log_capacity = 0,
                                                       bool allow_truncated = false) {
  return detail::optimizeLogged(prob, SqpParamRows(prob.GetBatch(), params), callbacks, detail::logDirs(params), log_capacity,
                                allow_truncated);
}
inline std::vector<sco::OptResults> OptimizeWithParams(TrajOptProb& prob,
                                                       const std::vector<sco::BasicTrustRegionSQPParameters>& params) {
  const std::vector<tb200_sqp_params> rows = SqpParamRows(prob.GetBatch(), params);
  const std::vector<std::string> dirs = detail::logDirs(params);
  if (!dirs.empty()) return detail::optimizeLogged(prob, rows, {}, dirs, 0, false);
  detail::setSqpParams(prob, rows);
  return detail::solveBatch(prob);
}

// The frames of every link of a RobotModel at joint values q: the arithmetic of the test oracle's Robot::fk (origin
// quaternion -> rotation, Rodrigues for a revolute joint, axis * q for a prismatic one, parent frame * origin * motion),
// restated here.  frames[j] is the frame the joint j creates (RobotModel::joints order): R row-major, then p.
struct Frame {
  double R[9];
  double p[3];
};
inline std::vector<Frame> RobotFK(const RobotModel& kin, const double* q) {
  auto mul = [](const Frame& a, const Frame& b) {
    Frame o{};
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += a.R[i * 3 + k] * b.R[k * 3 + j];
        o.R[i * 3 + j] = s;
      }
      o.p[i] = a.R[i * 3] * b.p[0] + a.R[i * 3 + 1] * b.p[1] + a.R[i * 3 + 2] * b.p[2] + a.p[i];
    }
    return o;
  };
  std::vector<Frame> f(kin.joints.size());
  for (size_t s = 0; s < kin.joints.size(); ++s) {
    const RobotModel::Joint& g = kin.joints[s];
    Frame t{};
    double w = g.origin.wxyz[0], x = g.origin.wxyz[1], y = g.origin.wxyz[2], z = g.origin.wxyz[3];
    const double n = std::sqrt(w * w + x * x + y * y + z * z);
    w /= n; x /= n; y /= n; z /= n;
    t.R[0] = 1 - 2 * (y * y + z * z); t.R[1] = 2 * (x * y - z * w);     t.R[2] = 2 * (x * z + y * w);
    t.R[3] = 2 * (x * y + z * w);     t.R[4] = 1 - 2 * (x * x + z * z); t.R[5] = 2 * (y * z - x * w);
    t.R[6] = 2 * (x * z - y * w);     t.R[7] = 2 * (y * z + x * w);     t.R[8] = 1 - 2 * (x * x + y * y);
    for (int i = 0; i < 3; ++i) t.p[i] = g.origin.xyz[i];
    if (g.type == TB200_JOINT_REVOLUTE) {
      const double a = q[g.q_index], c = std::cos(a), sn = std::sin(a), v = 1 - c;
      const double ax = g.axis[0], ay = g.axis[1], az = g.axis[2];
      Frame m{};
      m.R[0] = c + ax * ax * v;      m.R[1] = ax * ay * v - az * sn; m.R[2] = ax * az * v + ay * sn;
      m.R[3] = ay * ax * v + az * sn; m.R[4] = c + ay * ay * v;      m.R[5] = ay * az * v - ax * sn;
      m.R[6] = az * ax * v - ay * sn; m.R[7] = az * ay * v + ax * sn; m.R[8] = c + az * az * v;
      t = mul(t, m);
    } else if (g.type == TB200_JOINT_PRISMATIC) {
      Frame m{};
      m.R[0] = m.R[4] = m.R[8] = 1.0;
      for (int i = 0; i < 3; ++i) m.p[i] = g.axis[i] * q[g.q_index];
      t = mul(t, m);
    }
    f[s] = (g.parent < 0) ? t : mul(f[g.parent], t);
  }
  return f;
}
// Eigen::Quaterniond(Matrix3d) of a row-major rotation, (w, x, y, z): the trace branch and the largest-diagonal branch.
inline void RotToQuatWxyz(const double* m, double* q) {
  double t = m[0] + m[4] + m[8];
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m[7] - m[5]) * t;
    q[2] = (m[2] - m[6]) * t;
    q[3] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 3 + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
    q[1 + i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
  }
}

// trajopt::WriteCallback (file_write_callback.cpp) for the batch.  On creation it writes the header line: the joint names
// (here the child link of each moving joint, in column order), x,y,z,q_w,q_x,q_y,q_z, the cost names and the constraint
// names.  Every call then writes, per waypoint of the problem's x, a line of the joint values, then for every link of
// the model "<link>: " and ",x,y,z,qw,qx,qy,qz" of its frame (the reference iterates tesseract's TransformMap, an unordered
// map; here the links go in name order), then ",<cost>" per cost value and ",<violation>" per constraint value; and
// an empty line after the last waypoint.  Numbers go through operator<< as in the reference.  The problem index of the
// batch is not written: with several problems the blocks follow in call order.
inline Callback WriteCallback(std::shared_ptr<std::ofstream> file, std::shared_ptr<const RobotModel> kin,
                              const std::vector<std::string>& cost_names, const std::vector<std::string>& cnt_names) {
  if (!file->good()) std::fprintf(stderr, "ofstream passed to create callback not in 'good' state\n");
  std::vector<std::string> joint_names(kin->numJoints());
  for (const RobotModel::Joint& j : kin->joints)
    if (j.type != TB200_JOINT_FIXED && j.q_index >= 0 && j.q_index < kin->numJoints()) joint_names[j.q_index] = j.child_link;
  for (size_t i = 0; i < joint_names.size(); ++i) *file << (i ? "," : "") << joint_names[i];
  for (const char* s : {"x", "y", "z", "q_w", "q_x", "q_y", "q_z"}) *file << ',' << s;
  for (const auto& n : cost_names) *file << ',' << n;
  for (const auto& n : cnt_names) *file << ',' << n;
  *file << '\n' << std::flush;
  const int D = kin->numJoints();
  return [file, kin, D](TrajOptProb*, std::size_t, sco::OptResults& r) {
    std::map<std::string, size_t> links;  // name order
    for (size_t s = 0; s < kin->joints.size(); ++s) links.emplace(kin->joints[s].child_link, s);
    const size_t T = D ? r.x.size() / D : 0;
    for (size_t t = 0; t < T; ++t) {
      const double* q = r.x.data() + t * D;
      for (int j = 0; j < D; ++j) *file << (j ? "," : "") << q[j];
      const std::vector<Frame> fr = RobotFK(*kin, q);
      for (const auto& [name, s] : links) {
        double wxyz[4];
        RotToQuatWxyz(fr[s].R, wxyz);
        *file << name << ": ";
        for (double v : {fr[s].p[0], fr[s].p[1], fr[s].p[2], wxyz[0], wxyz[1], wxyz[2], wxyz[3]}) *file << ',' << v;
      }
      for (double c : r.cost_vals) *file << ',' << c;
      for (double c : r.cnt_viols) *file << ',' << c;
      *file << '\n';
    }
    *file << '\n' << std::flush;
  };
}
// ... for a problem: its robot model (pci.kin) and its object names (ObjectNames)
inline Callback WriteCallback(std::shared_ptr<std::ofstream> file, const TrajOptProb& prob) {
  std::vector<std::string> cost_names, cnt_names;
  ObjectNames(prob, cost_names, cnt_names);
  return WriteCallback(std::move(file), prob.flat().kin, cost_names, cnt_names);
}

// One problem of a multi-start solve (ProblemConstructionInfo::seeds_per_problem): its best seed and what every seed did.
struct MultiStartResult {
  int best = -1;                            // batch index of the best seed
  sco::OptResults result;                   // the best seed's results
  std::vector<sco::OptStatus> seed_status;  // status of every seed of the problem, in batch order
};

// Every problem of a multi-start batch, with the given parameters: the seeds are solved together (siblings stopped on the
// device when pci.stop_seeds_on_converged) and the best seed of each problem is selected on the device by the key of
// tb200_group_results (converged first, then the smallest constraint violation, then total cost, then index).
namespace detail {
inline std::vector<MultiStartResult> selectSeeds(TrajOptProb& prob, const std::vector<sco::OptResults>& seeds);
}
inline std::vector<MultiStartResult> OptimizeProblemMultiStart(TrajOptProb& prob, const tb200_sqp_params& params) {
  return detail::selectSeeds(prob, OptimizeWithParams(prob, params));
}
// ... with per-seed parameters (a parameter portfolio: the seeds of a problem may differ in their parameters as well as in
// their initial trajectory); params[b] for batch index b, as in OptimizeWithParams
inline std::vector<MultiStartResult> OptimizeProblemMultiStart(TrajOptProb& prob,
                                                              const std::vector<sco::BasicTrustRegionSQPParameters>& params) {
  return detail::selectSeeds(prob, OptimizeWithParams(prob, params));
}
inline std::vector<MultiStartResult> detail::selectSeeds(TrajOptProb& prob, const std::vector<sco::OptResults>& seeds) {
  const int G = prob.GetSeedsPerProblem(), NG = prob.GetBatch() / G;
  std::vector<int32_t> best(NG);
  tb200_group_results g{};
  g.best = best.data();
  if (tb200_fetch_group_results(prob.handle(), &g) != TB200_OK) throw std::runtime_error(tb200_last_error());
  std::vector<MultiStartResult> out(NG);
  for (int p = 0; p < NG; ++p) {
    out[p].best = best[p];
    out[p].result = seeds[best[p]];
    for (int k = 0; k < G; ++k) out[p].seed_status.push_back(seeds[p * G + k].status);
  }
  return out;
}
// ... with the problem description's own parameters (pci.opt_info)
inline std::vector<MultiStartResult> OptimizeProblemMultiStart(TrajOptProb& prob) {
  return OptimizeProblemMultiStart(prob, prob.sqpParams());
}

// tesseract::collision::CollisionCheckConfig, as the reference's tests pass it to checkTrajectory: the evaluator type
// (TB200_COLL_*), the longest valid segment length of the LVS types and the contact margin.
struct CollisionCheckConfig {
  int type = TB200_COLL_DISCRETE;
  double longest_valid_segment_length = 0.005;
  double contact_margin = 0.0;
};
using TrajArray = DblVec;  // one trajectory [T*D], row-major (tesseract's TrajArray is a T x D Eigen matrix)

// One trajectory's collision check.  Slots: one per waypoint (DISCRETE) or per step pair (the other types).
struct TrajectoryCheckResult {
  bool found = false;         // some slot has a contact (distance < contact_margin)
  int first_slot = -1;        // the first such slot
  double min_distance = 0;    // minimum over the slots (NaN when a distance is not finite)
  DblVec step_min_distance;   // per slot
  IntVec step_contacts;       // per slot: (sphere, obstacle, sub-state | sub-segment) triples in contact
};

// checkTrajectory for every trajectory of the batch (tb200_check_trajectories): trajs, one TrajArray per trajectory, or
// nullptr for the trajectories of the last solve (they stay on the device).
inline std::vector<TrajectoryCheckResult> checkTrajectories(TrajOptProb& prob, const CollisionCheckConfig& config,
                                                            const std::vector<TrajArray>* trajs = nullptr) {
  const size_t B = prob.GetBatch(), T = prob.GetNumSteps(), N = T * prob.GetNumDOF();
  DblVec x;
  if (trajs) {
    if (trajs->size() != B) throw std::runtime_error("checkTrajectories: one trajectory per problem of the batch is required");
    for (const TrajArray& t : *trajs) {
      if (t.size() != N) throw std::runtime_error("checkTrajectories: a trajectory has the wrong size");
      x.insert(x.end(), t.begin(), t.end());
    }
  }
  const size_t S = (config.type == TB200_COLL_DISCRETE) ? T : T - 1;
  DblVec smin(B * S), mind(B);
  std::vector<int32_t> cont(B * S), incoll(B), first(B);
  tb200_check_config c{};
  c.type = config.type;
  c.longest_valid_segment_length = config.longest_valid_segment_length;
  c.margin = config.contact_margin;
  tb200_check_results r{};
  r.step_min_distance = S ? smin.data() : nullptr;
  r.step_contacts = S ? cont.data() : nullptr;
  r.in_collision = incoll.data();
  r.first_slot = first.data();
  r.min_distance = mind.data();
  if (tb200_check_trajectories(prob.handle(), trajs ? x.data() : nullptr, &c, &r) != TB200_OK)
    throw std::runtime_error(tb200_last_error());
  std::vector<TrajectoryCheckResult> out(B);
  for (size_t b = 0; b < B; ++b) {
    out[b].found = incoll[b] != 0;
    out[b].first_slot = first[b];
    out[b].min_distance = mind[b];
    out[b].step_min_distance.assign(smin.begin() + b * S, smin.begin() + (b + 1) * S);
    out[b].step_contacts.assign(cont.begin() + b * S, cont.begin() + (b + 1) * S);
  }
  return out;
}

}  // namespace trajopt
}  // namespace trajopt_b200
