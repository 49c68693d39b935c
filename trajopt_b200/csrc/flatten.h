// The host half of problem creation: checks a tb200_problem_desc and flattens it into the tables the kernels read, the
// way trajopt::ConstructProblem / TermInfo::hatch do (trajopt/src/problem_description.cpp:410-542, 901-987, 1078-1176,
// 1197-1372, 1393-1493, 1714-1837).  Plain C++ without CUDA: a bad description gets the same answer with or without a
// device, and the flattened tables can be checked on any machine.
#pragma once
#include <algorithm>
#include <cmath>
#include <limits>
#include <string>
#include <utility>
#include <vector>

#include "../../include/trajopt_b200.h"
#include "device_types.cuh"

namespace tb200 {

// A description after the checks, the folding of the robot and the hatching of its terms: every table the library
// uploads for it, and the counts the layout of the kernels is planned from.
struct FlatProblem {
  // the robot, with the fixed segments nobody refers to folded into their children
  std::vector<DevSegment> segs;
  std::vector<DevSphere> spheres;           // [max(L, 1)]
  unsigned sphere_jmask[kMaxSpheres] = {};  // which trajectory columns move each sphere
  int qtype[kMaxDof] = {};                  // joint type per trajectory column
  int joint_seg[kMaxDof] = {};              // segment that carries trajectory column j
  std::vector<int> link_chain;              // [S][kMaxSeg + 1]: chain length, then the chain from the root to the segment
  // the cost and constraint objects in OptProb order (constraints: EQ first, then INEQ), and the (term, step) that
  // hatched each of them (costs, then constraints)
  std::vector<DevObj> cost_objs, cnt_objs;
  std::vector<std::pair<int, int>> obj_src;
  // copies of the CartPose, CartVel and collision objects for the evaluation kernel; collision objects in the order the
  // QP kernel meets them (costs first), which is also the order of their candidates
  std::vector<DevObj> cart_objs, vel_objs, coll_objs;
  std::vector<DevObj> sing_objs;  // avoid_singularity objects (one per step) for the evaluation kernel
  std::vector<DevJointTerm> joint_terms;
  std::vector<DevCartTerm> cart_terms;
  std::vector<int> fixed_vars;
  // quadratic objective of the state-independent costs: P = M + M' (osqp_interface.cpp:170-211), [N][2D + 1] and [N],
  // and the structurally non-zero offsets of its band (the kernels visit only these)
  std::vector<double> Pband, qlin;
  int n_band = 0, band_offs[32] = {};
  int n_cart_rows = 0, n_coll_cand = 0, max_rows = 0;
  bool has_vel = false, has_cast = false;
  int cast_cap = 0;  // active contacts (rows) a step pair of the continuous evaluator can hold
  int n_joint_objs = 0, joint_obj_idx[8] = {};  // positions of the joint-space objects in the (costs, cnts) list
  std::vector<SqpParams> sqp_rows;  // [B] optimizer parameters of trajectory b (sqp_per_traj[b], or sqp for every b)
};

namespace flat {

inline int refuse(std::string& msg, int code, const std::string& text) {
  msg = text;
  return code;
}

inline int check_groups(int B, int group_size, int group_stop, std::string& msg) {
  if (group_size < 0) return refuse(msg, TB200_ERR_INVALID, "group_size must be >= 0 (0 or 1: no groups)");
  if (group_size > 1 && B % group_size != 0)
    return refuse(msg, TB200_ERR_INVALID, "batch " + std::to_string(B) + " is not a multiple of group_size " + std::to_string(group_size));
  if (group_stop != 0 && group_stop != 1) return refuse(msg, TB200_ERR_INVALID, "group_stop must be 0 or 1");
  return TB200_OK;
}

inline SqpParams sqp_params(const tb200_sqp_params& s) {
  return SqpParams{s.improve_ratio_threshold, s.min_trust_box_size, s.min_approx_improve, s.min_approx_improve_frac,
                   s.trust_shrink_ratio, s.trust_expand_ratio, s.cnt_tolerance, s.max_merit_coeff_increases,
                   s.merit_coeff_increase_ratio, s.initial_merit_error_coeff, s.trust_box_size, s.max_iter,
                   s.max_qp_solver_failures, s.inflate_constraints_individually, 0, s.max_time};
}

// The parameters every trajectory of a batch of B runs under: rows[b] of a per-trajectory table, or `uniform` for every
// trajectory when there is none (rows NULL).
inline std::vector<SqpParams> sqp_rows(int B, const tb200_sqp_params& uniform, const tb200_sqp_params* rows) {
  std::vector<SqpParams> out(static_cast<size_t>(B), sqp_params(uniform));
  if (rows)
    for (int b = 0; b < B; ++b) out[b] = sqp_params(rows[b]);
  return out;
}

inline void quat_to_rot(const double* q, double* R) {
  double w = q[0], x = q[1], y = q[2], z = q[3];
  const double n = std::sqrt(w * w + x * x + y * y + z * z);
  w /= n; x /= n; y /= n; z /= n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}

// Joints that move segment s: the q_index bits of its chain.
inline unsigned joint_mask_of(const std::vector<DevSegment>& segs, int s) {
  unsigned m = 0;
  for (int a = s; a >= 0; a = segs[a].parent)
    if (segs[a].q_index >= 0) m |= 1u << segs[a].q_index;
  return m;
}

inline int check_args(const tb200_problem_desc& d, std::string& msg) {
  const int T = d.n_steps, D = d.robot.n_dof;
  if (T < 1 || T > TB200_MAX_STEPS) return refuse(msg, TB200_ERR_INVALID, "n_steps out of range");
  if (D < 1 || D > TB200_MAX_DOF) return refuse(msg, TB200_ERR_INVALID, "n_dof out of range");
  if (d.batch < 1) return refuse(msg, TB200_ERR_INVALID, "batch must be >= 1");
  if (int rc = check_groups(d.batch, d.group_size, d.group_stop, msg)) return rc;
  if (d.robot.n_segments < 1 || d.robot.n_segments > kMaxSeg) return refuse(msg, TB200_ERR_INVALID, "n_segments out of range");
  if (d.robot.n_spheres > kMaxSpheres) return refuse(msg, TB200_ERR_INVALID, "too many collision spheres");
  if (!d.init_traj) return refuse(msg, TB200_ERR_INVALID, "init_traj is required");
  if (d.n_terms < 0 || (d.n_terms > 0 && !d.terms)) return refuse(msg, TB200_ERR_INVALID, "terms is NULL with n_terms > 0");
  if (!d.robot.segments) return refuse(msg, TB200_ERR_INVALID, "robot.segments is NULL");
  if (!d.robot.lower || !d.robot.upper) return refuse(msg, TB200_ERR_INVALID, "robot joint limits are NULL");
  if (d.robot.n_spheres < 0 || (d.robot.n_spheres > 0 && !d.robot.spheres))
    return refuse(msg, TB200_ERR_INVALID, "robot.spheres is NULL with n_spheres > 0");
  if (d.n_fixed_timesteps < 0 || (d.n_fixed_timesteps > 0 && !d.fixed_timesteps))
    return refuse(msg, TB200_ERR_INVALID, "fixed_timesteps is NULL with n_fixed_timesteps > 0");
  if (d.n_fixed_dofs < 0 || (d.n_fixed_dofs > 0 && !d.fixed_dofs))
    return refuse(msg, TB200_ERR_INVALID, "fixed_dofs is NULL with n_fixed_dofs > 0");
  if (d.n_obstacles < 0 || (d.n_obstacles > 0 && !d.obstacles))
    return refuse(msg, TB200_ERR_INVALID, "obstacles is NULL with n_obstacles > 0");
  if (d.n_cart_targets < 0 || (d.n_cart_targets > 0 && !d.cart_targets))
    return refuse(msg, TB200_ERR_INVALID, "cart_targets is NULL with n_cart_targets > 0");
  return TB200_OK;
}

// The segments, spheres and joint tables.  Fixed segments nobody refers to (no collision sphere, no Cartesian term) are
// folded into their children: child.origin <- fixed.origin * child.origin.  The kernels then carry fewer frames per
// waypoint (shared memory of the evaluation kernel: 12 doubles per frame and waypoint).  remap: the kept index of every
// segment of the description (-1: folded).
inline int fold_robot(const tb200_problem_desc& d, FlatProblem& F, std::vector<int>& remap, std::string& msg) {
  const int D = d.robot.n_dof, S = d.robot.n_segments, L = d.robot.n_spheres;
  std::vector<DevSegment> segs(S);
  for (int s = 0; s < S; ++s) {
    const tb200_segment& g = d.robot.segments[s];
    if (g.parent >= s) return refuse(msg, TB200_ERR_INVALID, "segments must be topologically ordered");
    if (g.joint_type != TB200_JOINT_FIXED && (g.q_index < 0 || g.q_index >= D)) return refuse(msg, TB200_ERR_INVALID, "bad q_index");
    segs[s].parent = g.parent; segs[s].joint_type = g.joint_type; segs[s].q_index = g.joint_type == TB200_JOINT_FIXED ? -1 : g.q_index;
    quat_to_rot(g.origin_wxyz, segs[s].R);
    for (int i = 0; i < 3; ++i) { segs[s].p[i] = g.origin_xyz[i]; segs[s].axis[i] = g.axis[i]; }
    if (g.joint_type != TB200_JOINT_FIXED) F.qtype[g.q_index] = g.joint_type;
  }
  std::vector<char> used(S, 0);
  for (int s = 0; s < L; ++s) {
    const int g = d.robot.spheres[s].segment;
    if (g < 0 || g >= S) return refuse(msg, TB200_ERR_INVALID, "sphere attached to a bad segment");
    used[g] = 1;
  }
  for (int k = 0; k < d.n_terms; ++k)
    if ((d.terms[k].kind == TB200_TERM_CART_POSE || d.terms[k].kind == TB200_TERM_CART_VEL ||
         d.terms[k].kind == TB200_TERM_AVOID_SINGULARITY) &&
        d.terms[k].link >= 0 && d.terms[k].link < S)
      used[d.terms[k].link] = 1;
  remap.assign(S, -1);
  std::vector<DevSegment> acc(S);  // transform from the nearest kept ancestor's frame to this (folded) segment
  for (int s = 0; s < S; ++s) {
    DevSegment g = segs[s];
    const int par = g.parent;
    if (par >= 0 && remap[par] < 0) {  // parent was folded: compose its accumulated origin in front of ours
      const DevSegment& a = acc[par];
      double R[9], pp[3];
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) R[i * 3 + j] = a.R[i * 3] * g.R[j] + a.R[i * 3 + 1] * g.R[3 + j] + a.R[i * 3 + 2] * g.R[6 + j];
        pp[i] = a.R[i * 3] * g.p[0] + a.R[i * 3 + 1] * g.p[1] + a.R[i * 3 + 2] * g.p[2] + a.p[i];
      }
      for (int i = 0; i < 9; ++i) g.R[i] = R[i];
      for (int i = 0; i < 3; ++i) g.p[i] = pp[i];
      g.parent = a.parent;  // nearest kept ancestor (original index) or -1
    }
    if (g.joint_type == TB200_JOINT_FIXED && !used[s]) {
      acc[s] = g;  // folded: remembered for its children
    } else {
      remap[s] = static_cast<int>(F.segs.size());
      g.parent = (g.parent >= 0) ? remap[g.parent] : -1;
      F.segs.push_back(g);
    }
  }
  F.spheres.assign(std::max(L, 1), DevSphere{});
  for (int s = 0; s < L; ++s) {
    const tb200_sphere& sp = d.robot.spheres[s];
    F.spheres[s].segment = remap[sp.segment]; F.spheres[s].r = sp.radius;
    for (int i = 0; i < 3; ++i) F.spheres[s].c[i] = sp.center[i];
    F.sphere_jmask[s] = joint_mask_of(F.segs, F.spheres[s].segment);
  }
  const int Sk = static_cast<int>(F.segs.size());
  F.link_chain.assign(static_cast<size_t>(Sk) * (kMaxSeg + 1), 0);
  for (int sg = 0; sg < Sk; ++sg) {
    if (F.segs[sg].q_index >= 0) F.joint_seg[F.segs[sg].q_index] = sg;
    std::vector<int> up;
    for (int a = sg; a >= 0; a = F.segs[a].parent) up.push_back(a);
    int* c = F.link_chain.data() + static_cast<size_t>(sg) * (kMaxSeg + 1);
    c[0] = static_cast<int>(up.size());
    for (size_t k = 0; k < up.size(); ++k) c[1 + k] = up[up.size() - 1 - k];
  }
  return TB200_OK;
}

// The objects of the three lists (costs, EQ constraints, INEQ constraints) while the terms are hatched: each is appended
// together with its source, and the CartPose, CartVel and collision objects are also remembered by (list, index).
struct Lists {
  enum Id { COST = 0, EQ = 1, INEQ = 2 };
  using Ref = std::pair<Id, int>;
  std::vector<DevObj> obj[3];
  std::vector<std::pair<int, int>> src[3];
  std::vector<Ref> cart, vel, coll, sing;
  Ref add(Id l, const DevObj& o, int term, int step) {
    obj[l].push_back(o);
    src[l].push_back({term, step});
    return {l, static_cast<int>(obj[l].size()) - 1};
  }
};

inline int hatch_terms(const tb200_problem_desc& d, const std::vector<int>& remap, FlatProblem& F, Lists& lists, std::string& msg) {
  const int T = d.n_steps, D = d.robot.n_dof, L = d.robot.n_spheres, O = d.n_obstacles;
  bool has_discrete = false;
  for (int k = 0; k < d.n_terms; ++k) {
    const tb200_term& tm = d.terms[k];
    if (tm.role != TB200_ROLE_COST && tm.role != TB200_ROLE_CNT) return refuse(msg, TB200_ERR_INVALID, "term role must be COST or CNT");
    const bool is_cnt = tm.role == TB200_ROLE_CNT;
    DevObj o{};
    o.is_cnt = is_cnt;
    if (tm.kind == TB200_TERM_JOINT_POS || tm.kind == TB200_TERM_JOINT_VEL || tm.kind == TB200_TERM_JOINT_ACC) {
      o.order = tm.kind - TB200_TERM_JOINT_POS;
      o.first = tm.first_step;
      o.n_steps = tm.last_step - tm.first_step + 1 - o.order;
      if (tm.first_step < 0 || tm.last_step >= T) return refuse(msg, TB200_ERR_INVALID, "joint term steps outside the trajectory");
      if (o.n_steps <= 0) return refuse(msg, TB200_ERR_INVALID, "joint term: trajectory is too short");
      DevJointTerm jt{};
      bool zero_tol = true;
      for (int j = 0; j < D; ++j) {
        jt.coeffs[j] = tm.coeffs[j]; jt.targets[j] = tm.targets[j]; jt.upper[j] = tm.upper_tols[j]; jt.lower[j] = tm.lower_tols[j];
        zero_tol = zero_tol && std::fabs(tm.upper_tols[j]) < 1e-5 && std::fabs(tm.lower_tols[j]) < 1e-5;
      }
      o.term = static_cast<int>(F.joint_terms.size());
      F.joint_terms.push_back(jt);
      if (!is_cnt) {
        o.kind = zero_tol ? OBJ_JOINT_EQ_COST : OBJ_JOINT_INEQ_COST;
        o.n_rows = zero_tol ? 0 : 2 * o.n_steps * D;
        lists.add(Lists::COST, o, k, tm.first_step);
      } else {
        o.kind = zero_tol ? OBJ_JOINT_EQ_CNT : OBJ_JOINT_INEQ_CNT;
        o.n_rows = (zero_tol ? 1 : 2) * o.n_steps * D;
        lists.add(zero_tol ? Lists::EQ : Lists::INEQ, o, k, tm.first_step);
      }
      F.max_rows += o.n_rows;
    } else if (tm.kind == TB200_TERM_CART_POSE) {
      if (tm.first_step < 0 || tm.first_step >= T) return refuse(msg, TB200_ERR_INVALID, "cart_pose timestep outside the trajectory");
      if (tm.link < 0 || tm.link >= d.robot.n_segments) return refuse(msg, TB200_ERR_INVALID, "cart_pose link out of range");
      if (tm.target_slot >= d.n_cart_targets) return refuse(msg, TB200_ERR_INVALID, "cart_pose target_slot out of range");
      DevCartTerm ct{};
      quat_to_rot(tm.source_offset + 3, ct.src_R);
      for (int i = 0; i < 3; ++i) ct.src_p[i] = tm.source_offset[i];
      for (int i = 0; i < 7; ++i) ct.tgt[i] = tm.target_pose[i];
      for (int i = 0; i < 3; ++i)
        if (std::fabs(tm.pos_coeffs[i]) > 1e-5) { ct.idx[ct.n_idx] = i; ct.coeff[ct.n_idx++] = tm.pos_coeffs[i]; }
      for (int i = 0; i < 3; ++i)
        if (std::fabs(tm.rot_coeffs[i]) > 1e-5) { ct.idx[ct.n_idx] = 3 + i; ct.coeff[ct.n_idx++] = tm.rot_coeffs[i]; }
      o.kind = OBJ_CART_POSE;
      o.first = tm.first_step;
      o.link = remap[tm.link];
      o.target_slot = tm.target_slot;
      o.term = static_cast<int>(F.cart_terms.size());
      o.src_off = F.n_cart_rows;
      o.n_rows = ct.n_idx;
      F.cart_terms.push_back(ct);
      F.n_cart_rows += ct.n_idx;
      F.max_rows += ct.n_idx;
      lists.cart.push_back(lists.add(is_cnt ? Lists::EQ : Lists::COST, o, k, tm.first_step));
    } else if (tm.kind == TB200_TERM_COLLISION) {
      if (tm.evaluator_type < TB200_COLL_DISCRETE || tm.evaluator_type > TB200_COLL_LVS_CONTINUOUS)
        return refuse(msg, TB200_ERR_INVALID, "unknown collision evaluator type");
      if (L == 0 || O == 0) return refuse(msg, TB200_ERR_INVALID, "collision term needs robot spheres and obstacles");
      if (tm.n_fixed_steps < 0 || tm.n_fixed_steps > 8) return refuse(msg, TB200_ERR_INVALID, "collision term: n_fixed_steps outside [0, 8]");
      const bool cast = tm.evaluator_type != TB200_COLL_DISCRETE;
      if (cast && tm.evaluator_type != TB200_COLL_CONTINUOUS && !(tm.longest_valid_segment_length > 0.0))
        return refuse(msg, TB200_ERR_INVALID, "longest_valid_segment_length must be positive");
      if ((cast && has_discrete) || (!cast && F.has_cast))
        return refuse(msg, TB200_ERR_UNSUPPORTED, "discrete and continuous collision terms in one problem are not supported");
      (cast ? F.has_cast : has_discrete) = true;
      // discrete: one object per non-fixed step (problem_description.cpp:1762-1775, 1824-1833); continuous: one per
      // step pair [first, last) with the expression type taken from the fixed steps (:1714-1760, 1776-1819)
      for (int t = tm.first_step; cast ? t < tm.last_step : t <= tm.last_step; ++t) {
        bool fixed = false, next_fixed = false;
        for (int f = 0; f < tm.n_fixed_steps; ++f) {
          fixed |= tm.fixed_steps[f] == t;
          next_fixed |= tm.fixed_steps[f] == t + 1;
        }
        if (!cast && fixed) continue;
        if (t < 0 || t + (cast ? 1 : 0) >= T) return refuse(msg, TB200_ERR_INVALID, "collision step outside the trajectory");
        DevObj c = o;
        c.kind = cast ? OBJ_COLL_CAST : OBJ_COLL;
        c.first = t;
        c.n_rows = cast ? F.cast_cap : L * O;  // continuous: room for cast_cap active contacts of the step pair
        c.coeff = tm.coeff; c.margin = tm.margin; c.buffer = tm.margin_buffer;
        // (two adjacent fixed steps take the START_FIXED_END_FREE branch: the reference's throw is unreachable)
        // LVS_DISCRETE: a discrete test at every state of the sub-trajectory instead of a swept one per sub-segment
        if (cast)
          c.cast_flags = (fixed ? CAST_START_FIXED : 0) | ((!fixed && next_fixed) ? CAST_END_FIXED : 0) |
                         (tm.evaluator_type == TB200_COLL_LVS_DISCRETE ? CAST_LVS_DISCRETE : 0);
        c.lvs = (tm.evaluator_type == TB200_COLL_CONTINUOUS) ? std::numeric_limits<double>::max() : tm.longest_valid_segment_length;
        lists.coll.push_back(lists.add(is_cnt ? Lists::INEQ : Lists::COST, c, k, t));
      }
    } else if (tm.kind == TB200_TERM_CART_VEL) {
      // CartVelTermInfo::hatch (problem_description.cpp:1011-1057): one object per step pair (t, t+1)
      if (tm.link < 0 || tm.link >= d.robot.n_segments) return refuse(msg, TB200_ERR_INVALID, "cart_vel link out of range");
      for (int t = tm.first_step; t <= tm.last_step; ++t) {
        if (t < 0 || t + 1 >= T) return refuse(msg, TB200_ERR_INVALID, "cart_vel: step pair beyond the trajectory");
        DevObj c = o;
        c.kind = OBJ_CART_VEL;
        c.first = t;
        c.link = remap[tm.link];
        c.src_off = F.n_cart_rows;
        c.n_rows = 6;
        c.joint_mask = static_cast<int>(joint_mask_of(F.segs, c.link));
        c.lvs = tm.max_displacement;
        F.n_cart_rows += 6;
        F.max_rows += 6;
        F.has_vel = true;
        lists.vel.push_back(lists.add(is_cnt ? Lists::INEQ : Lists::COST, c, k, t));
      }
    } else if (tm.kind == TB200_TERM_AVOID_SINGULARITY) {
      // AvoidSingularityTermInfo::hatch (problem_description.cpp:1900-1939): one object per step over its D joints, an
      // ABS cost or an INEQ constraint; fixed timesteps are not skipped.  (The reference's defaults first_step =
      // last_step = -1 would index step -1: refused here.)
      if (tm.link < 0 || tm.link >= d.robot.n_segments) return refuse(msg, TB200_ERR_INVALID, "avoid_singularity link out of range");
      if (tm.first_step < 0 || tm.last_step >= T || tm.first_step > tm.last_step)
        return refuse(msg, TB200_ERR_INVALID, "avoid_singularity steps outside the trajectory");
      if (!std::isfinite(tm.lambda) || tm.lambda < 0.0)
        return refuse(msg, TB200_ERR_INVALID, "avoid_singularity lambda must be finite and >= 0");
      for (int t = tm.first_step; t <= tm.last_step; ++t) {
        DevObj c = o;
        c.kind = OBJ_SINGULARITY;
        c.first = t;
        c.link = remap[tm.link];
        c.src_off = F.n_cart_rows;
        c.n_rows = 1;
        c.coeff = tm.coeffs[0];
        c.margin = tm.lambda;
        F.n_cart_rows += 1;
        F.max_rows += 1;
        lists.sing.push_back(lists.add(is_cnt ? Lists::INEQ : Lists::COST, c, k, t));
      }
    } else {
      return refuse(msg, TB200_ERR_INVALID, "unknown term kind");
    }
  }
  return TB200_OK;
}

// The object lists in OptProb order and the evaluation kernel's copies.  The collision candidates are laid out in the
// kernel order of the collision objects (src_off), and kernel_slot is where the evaluation kernel leaves an object's value.
inline void order_objects(Lists& lists, FlatProblem& F) {
  F.cost_objs = lists.obj[Lists::COST];
  F.cnt_objs = lists.obj[Lists::EQ];
  F.cnt_objs.insert(F.cnt_objs.end(), lists.obj[Lists::INEQ].begin(), lists.obj[Lists::INEQ].end());
  for (const auto& s : lists.src) F.obj_src.insert(F.obj_src.end(), s.begin(), s.end());
  const int n_eq = static_cast<int>(lists.obj[Lists::EQ].size());
  auto index_of = [&](Lists::Ref r) { return r.first == Lists::INEQ ? n_eq + r.second : r.second; };
  auto object = [&](Lists::Ref r) -> DevObj& { return r.first == Lists::COST ? F.cost_objs[r.second] : F.cnt_objs[index_of(r)]; };
  auto copy = [&](Lists::Ref r) {
    DevObj o = object(r);
    o.list_index = index_of(r);
    return o;
  };
  for (Lists::Ref r : lists.cart) F.cart_objs.push_back(copy(r));
  for (Lists::Ref r : lists.vel) F.vel_objs.push_back(copy(r));
  for (Lists::Ref r : lists.sing) F.sing_objs.push_back(copy(r));
  for (const bool costs : {true, false})
    for (Lists::Ref r : lists.coll) {
      if (costs != (r.first == Lists::COST)) continue;
      DevObj& o = object(r);
      o.src_off = F.n_coll_cand;
      o.kernel_slot = static_cast<int>(F.coll_objs.size());
      F.n_coll_cand += o.n_rows;
      F.coll_objs.push_back(copy(r));
    }
  F.max_rows += F.n_coll_cand;
}

inline int fixed_variables(const tb200_problem_desc& d, FlatProblem& F, std::string& msg) {
  const int T = d.n_steps, D = d.robot.n_dof;
  for (int k = 0; k < d.n_fixed_timesteps; ++k) {
    const int t = d.fixed_timesteps[k];
    if (t < 0 || t >= T) return refuse(msg, TB200_ERR_INVALID, "Fixed timestep index is outside the bounds of the initial trajectory.");
    for (int j = 0; j < D; ++j) F.fixed_vars.push_back(t * D + j);
  }
  for (int k = 0; k < d.n_fixed_dofs; ++k) {
    const int j = d.fixed_dofs[k];
    if (j < 0 || j >= D) return refuse(msg, TB200_ERR_INVALID, "DOF(aka Joint) indice is greater than the number of DOF available.");
    for (int t = 0; t < T; ++t) {
      bool skip = false;
      for (int f = 0; f < d.n_fixed_timesteps; ++f) skip |= d.fixed_timesteps[f] == t;
      if (!skip) F.fixed_vars.push_back(t * D + j);
    }
  }
  F.max_rows = std::max(F.max_rows + static_cast<int>(F.fixed_vars.size()), 1);
  return TB200_OK;
}

inline void quadratic_objective(int T, int D, FlatProblem& F) {
  const int N = T * D, W = 2 * D + 1;
  F.Pband.assign(static_cast<size_t>(N) * W, 0.0);
  F.qlin.assign(N, 0.0);
  for (const DevObj& o : F.cost_objs) {
    if (o.kind != OBJ_JOINT_EQ_COST) continue;
    static const double wst[3][3] = {{1, 0, 0}, {-1, 1, 0}, {1, -2, 1}};
    const DevJointTerm& jt = F.joint_terms[o.term];
    for (int t = o.first; t < o.first + o.n_steps; ++t)
      for (int j = 0; j < D; ++j)
        for (int a = 0; a <= o.order; ++a) {
          const int ia = (t + a) * D + j;
          F.qlin[ia] += -2.0 * jt.coeffs[j] * jt.targets[j] * wst[o.order][a];
          for (int bb = 0; bb <= a; ++bb) {
            const int ib = (t + bb) * D + j;
            F.Pband[static_cast<size_t>(ia) * W + (ia - ib)] += 2.0 * jt.coeffs[j] * wst[o.order][a] * wst[o.order][bb];
          }
        }
  }
  for (int k = 0; k < W; ++k) {
    bool nz = false;
    for (int i = k; i < N && !nz; ++i) nz = F.Pband[static_cast<size_t>(i) * W + k] != 0.0;
    if (nz) F.band_offs[F.n_band++] = k;
  }
}

}  // namespace flat

// Checks the description d and flattens it into F.  Returns TB200_OK or an error code with its message in msg: the first
// fault in the order arguments, robot, terms (in their order), fixed variables, then the kernels' limits on joint-space
// objects and obstacles.
inline int flatten(const tb200_problem_desc& d, FlatProblem& F, std::string& msg) {
  if (int rc = flat::check_args(d, msg)) return rc;
  std::vector<int> remap;
  if (int rc = flat::fold_robot(d, F, remap, msg)) return rc;
  F.cast_cap = tb200inl_cast_rows_per_pair(&d);
  flat::Lists lists;
  if (int rc = flat::hatch_terms(d, remap, F, lists, msg)) return rc;
  flat::order_objects(lists, F);
  if (int rc = flat::fixed_variables(d, F, msg)) return rc;
  flat::quadratic_objective(d.n_steps, d.robot.n_dof, F);
  int idx = 0;
  for (const auto* objs : {&F.cost_objs, &F.cnt_objs})
    for (const DevObj& o : *objs) {
      if (o.kind <= OBJ_JOINT_INEQ_CNT) {
        if (F.n_joint_objs < 8) F.joint_obj_idx[F.n_joint_objs] = idx;
        F.n_joint_objs++;
      }
      ++idx;
    }
  if (F.n_joint_objs > 8) return flat::refuse(msg, TB200_ERR_UNSUPPORTED, "more than 8 joint-space cost/constraint objects");
  if (d.n_obstacles > 64) return flat::refuse(msg, TB200_ERR_UNSUPPORTED, "more than 64 obstacle spheres per trajectory");
  F.sqp_rows = flat::sqp_rows(d.batch, d.sqp, d.sqp_per_traj);
  return TB200_OK;
}

}  // namespace tb200
