// Host side of the C ABI (include/trajopt_b200.h): validates and flattens the problem description the
// way trajopt::ConstructProblem / TermInfo::hatch do (trajopt/src/problem_description.cpp:410-542,
// 901-987, 1078-1176, 1197-1372, 1393-1493, 1714-1837), owns the device buffers, and drives the
// batched trust-region SQP (trajopt_sco/src/optimizers.cpp:699-991): one launch of eval_convexify_decide_kernel
// (first evaluation + convexification of every trajectory) and one persistent launch of solve_kernel, which runs
// every trajectory's QP subproblems, merit evaluations, re-convexifications and accept/shrink/penalty decisions.
// CUDA only: every entry point fails with TB200_ERR_CUDA / TB200_ERR_NO_DEVICE when no device is usable.
#include <cuda_runtime.h>
#include <math_constants.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "../../include/trajopt_b200.h"
#include "check_kernel.cuh"
#include "eval_kernel.cuh"
#include "solve_kernel.cuh"
#include "kernels.h"

using namespace tb200;

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CK(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (call);                                                                          \
    if (e_ != cudaSuccess) return fail(TB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaError_t alloc(size_t count) {
    n = count;
    if (count == 0) count = 1;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e == cudaSuccess) e = cudaMemset(p, 0, count * sizeof(T));
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
  }
};

int checkGroups(int B, int group_size, int group_stop) {
  if (group_size < 0) return fail(TB200_ERR_INVALID, "group_size must be >= 0 (0 or 1: no groups)");
  if (group_size > 1 && B % group_size != 0)
    return fail(TB200_ERR_INVALID, "batch " + std::to_string(B) + " is not a multiple of group_size " + std::to_string(group_size));
  if (group_stop != 0 && group_stop != 1) return fail(TB200_ERR_INVALID, "group_stop must be 0 or 1");
  return TB200_OK;
}
// G = 0 and G = 1 are both "no groups": every trajectory is its own group and nothing is stopped
void setGroups(DevProblem& dp, int group_size, int group_stop) {
  dp.group_size = std::max(group_size, 1);
  dp.group_stop = dp.group_size > 1 ? group_stop : 0;
}

void quatToRot(const double* q, double* R) {
  double w = q[0], x = q[1], y = q[2], z = q[3];
  const double n = std::sqrt(w * w + x * x + y * y + z * z);
  w /= n; x /= n; y /= n; z /= n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}
}  // namespace

struct tb200_problem {
  int device = 0;
  DevProblem dp{};
  EvalExtra ex{};
  tb200_layout layout{};
  int B = 0, T = 0, D = 0, N = 0;
  size_t eval_smem = 0, qp_smem = 0, solve_smem = 0;
  int n_sm = 132;  // H100 SXM; replaced by the device's own count at problem creation
  int quantum = 3;  // SQP steps a CTA runs of a trajectory before it looks for a more urgent one (TB200_QUANTUM overrides)
  cudaStream_t stream = nullptr;
  tb200_timing timing{};
  // host copies of the flattened description
  std::vector<DevObj> cost_objs, cnt_objs, cart_objs, coll_objs, vel_objs;
  std::vector<std::pair<int, int>> obj_src;  // per object (costs, then constraints): the term that hatched it, its step
  // SQP iteration log: the setting of the next solve, and the buffers of the last one (log_solved: it ran with the log)
  int log_cap_next = 0, log_with_x_next = 0;
  bool log_solved = false;
  DevBuf<double> log;
  DevBuf<int> log_len, log_dropped;
  bool pair_rows = false;  // QP rows span two waypoints (CartVel, continuous collision): 2*D coefficients per row
  // device storage
  DevBuf<DevSegment> segs;
  DevBuf<DevSphere> spheres;
  DevBuf<double> lower, upper, Pband, qlin, init_traj, cart_targets, obstacles;
  DevBuf<DevObj> d_cost_objs, d_cnt_objs, d_cart_objs, d_coll_objs, d_vel_objs;
  DevBuf<DevJointTerm> joint_terms;
  DevBuf<DevCartTerm> cart_terms;
  DevBuf<int> fixed_vars;
  DevBuf<double> x, new_x, trust, merit_coeffs, cost_vals, cnt_viols, new_cost_vals, new_cnt_viols, model_cost_vals,
      model_cnt_viols, cart_err, cart_jac, coll_rows, rows, ws_x, ws_yb, scratch, ws_rho, x_tmp, trust_tmp, dbg, trace, factor_g, cast_scratch, soa;
  DevBuf<unsigned long long> sched_timers, clock_start;
  DevBuf<int> sched_state, sqp_top, ended_by, group_done, qp_paths;
  // the best seed of every group (group_select_kernel): [NG] index, status, n_converged, total cost; [NG][N] its x
  DevBuf<int> g_best, g_status, g_n_converged;
  DevBuf<double> g_total_cost, g_x;
  int solved_group_size = 0;  // group_size of the last solve (0: no solve yet)
  bool selected = false;      // g_* hold the selection of the last solve
  // results of tb200_check_trajectories: [B][T] per slot (minimum, contacts, argmin x3), [B] per trajectory; allocated
  // by the first check
  DevBuf<double> chk_slot_min, chk_min;
  DevBuf<int> chk_slot_contacts, chk_slot_argmin, chk_in_collision, chk_first;
  DevBuf<unsigned long long> coll_mask;
  DevBuf<int> status, sqp_iter, merit_round, qp_failures, qp_status, cur_buf, n_qp_solves, n_func_evals, n_admm_iters,
      active_count, row_ints, lists, ws_meta, tmp_iters, tmp_polish, trace_len, qp_done, lvs_overflow, link_chain, work_counter;
  int eval_grid = 1;  // CTAs of a stand-alone evaluation launch: what fits the device at once (persistent CTAs)
  int cast_cap = TB200_MIN_CAST_ROWS_PER_PAIR;  // active contacts (rows) a step pair of the continuous evaluator can hold
  size_t factor_grid = 0;  // CTAs that own a region of factor_g (0: the factor lives in shared memory)
  std::vector<cudaEvent_t> events;
  ~tb200_problem() {
    for (auto e : events) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
    segs.release(); spheres.release(); lower.release(); upper.release(); Pband.release(); qlin.release();
    init_traj.release(); cart_targets.release(); obstacles.release(); d_cost_objs.release(); d_cnt_objs.release();
    d_cart_objs.release(); d_coll_objs.release(); d_vel_objs.release(); joint_terms.release(); cart_terms.release(); fixed_vars.release();
    x.release(); new_x.release(); trust.release(); merit_coeffs.release(); cost_vals.release(); cnt_viols.release();
    new_cost_vals.release(); new_cnt_viols.release(); model_cost_vals.release(); model_cnt_viols.release();
    cart_err.release(); cart_jac.release(); coll_rows.release(); rows.release(); ws_x.release(); ws_yb.release();
    scratch.release(); ws_rho.release(); dbg.release(); trace.release(); trace_len.release(); factor_g.release(); cast_scratch.release(); soa.release(); lvs_overflow.release(); link_chain.release(); work_counter.release(); qp_done.release(); sched_state.release(); sched_timers.release(); clock_start.release(); sqp_top.release(); ended_by.release(); group_done.release(); qp_paths.release(); g_best.release(); g_status.release(); g_n_converged.release(); g_total_cost.release(); g_x.release(); x_tmp.release(); trust_tmp.release(); coll_mask.release(); status.release();
    sqp_iter.release(); merit_round.release(); qp_failures.release(); qp_status.release(); cur_buf.release();
    n_qp_solves.release(); n_func_evals.release(); n_admm_iters.release(); active_count.release(); row_ints.release();
    lists.release(); ws_meta.release(); tmp_iters.release(); tmp_polish.release();
    chk_slot_min.release(); chk_min.release(); chk_slot_contacts.release(); chk_slot_argmin.release(); chk_in_collision.release();
    chk_first.release();
    log.release(); log_len.release(); log_dropped.release();
  }
};

extern "C" {

const char* tb200_version(void) { return "trajopt_b200 0.5 (sm_90a)"; }
const char* tb200_last_error(void) { return g_err.c_str(); }

void tb200_default_sqp_params(tb200_sqp_params* p) {  // optimizers.hpp:92-135
  p->improve_ratio_threshold = 0.25;
  p->min_trust_box_size = 1e-4;
  p->min_approx_improve = 1e-4;
  p->min_approx_improve_frac = -1.7976931348623157e308;
  p->max_iter = 50;
  p->max_qp_solver_failures = 3;
  p->trust_shrink_ratio = 0.1;
  p->trust_expand_ratio = 1.5;
  p->cnt_tolerance = 1e-4;
  p->max_merit_coeff_increases = 5;
  p->merit_coeff_increase_ratio = 10;
  p->initial_merit_error_coeff = 10;
  p->trust_box_size = 0.1;
  p->inflate_constraints_individually = 1;
  p->reserved = 0;
  p->max_time = std::numeric_limits<double>::max();  // no time limit
}
void tb200_osqp_order_qp_settings(tb200_qp_settings* s) {
  tb200_default_qp_settings(s);
  s->early_polish_every = 0;  // polish only after ADMM converged, as OSQP does
  s->early_polish_from = 0;
}
// The reference's OSQPSettings (osqp_interface.cpp:78-90 over osqp_set_default_settings) plus two choices that are NOT
// OSQP's (DESIGN.md section 6): a fixed adaptive_rho_interval (D0: OSQP's default is wall-clock based), and the early
// VERIFIED polish (O1: early_polish_every / early_polish_from = 25) - same minimiser, ~40 % fewer ADMM iterations;
// tb200_osqp_order_qp_settings turns it off.  Two more deviations are not settings but how the QP step works: the warm
// start from the ADMM duals (D1) and the verified polish (D2).
void tb200_default_qp_settings(tb200_qp_settings* s) {
  s->rho = 0.1; s->sigma = 1e-6; s->alpha = 1.6;
  s->eps_abs = 1e-4; s->eps_rel = 1e-6;
  s->eps_prim_inf = 1e-4; s->eps_dual_inf = 1e-4;
  s->delta = 1e-6; s->adaptive_rho_tolerance = 5.0;
  s->max_iter = 8192; s->scaling = 10; s->check_termination = 25;
  s->adaptive_rho = 1; s->adaptive_rho_interval = 50;
  s->polishing = 1; s->polish_refine_iter = 3; s->warm_starting = 1;
  s->early_polish_every = 25; s->early_polish_from = 25;
}

int tb200_problem_create(const tb200_problem_desc* d, int device, tb200_problem** out) {
  if (!d || !out) return fail(TB200_ERR_INVALID, "null argument");
  *out = nullptr;
  // (the description is checked and flattened first - pure host work, so that a bad description gets the same
  // error with or without a device - and only then the device is touched)
  const int T = d->n_steps, D = d->robot.n_dof, B = d->batch, N = T * D;
  if (T < 1 || T > TB200_MAX_STEPS) return fail(TB200_ERR_INVALID, "n_steps out of range");
  if (D < 1 || D > TB200_MAX_DOF) return fail(TB200_ERR_INVALID, "n_dof out of range");
  if (B < 1) return fail(TB200_ERR_INVALID, "batch must be >= 1");
  if (int rc = checkGroups(B, d->group_size, d->group_stop)) return rc;
  if (d->robot.n_segments < 1 || d->robot.n_segments > kMaxSeg) return fail(TB200_ERR_INVALID, "n_segments out of range");
  if (d->robot.n_spheres > kMaxSpheres) return fail(TB200_ERR_INVALID, "too many collision spheres");
  if (!d->init_traj) return fail(TB200_ERR_INVALID, "init_traj is required");
  if (d->n_terms < 0 || (d->n_terms > 0 && !d->terms)) return fail(TB200_ERR_INVALID, "terms is NULL with n_terms > 0");
  if (!d->robot.segments) return fail(TB200_ERR_INVALID, "robot.segments is NULL");
  if (!d->robot.lower || !d->robot.upper) return fail(TB200_ERR_INVALID, "robot joint limits are NULL");
  if (d->robot.n_spheres < 0 || (d->robot.n_spheres > 0 && !d->robot.spheres))
    return fail(TB200_ERR_INVALID, "robot.spheres is NULL with n_spheres > 0");
  if (d->n_fixed_timesteps < 0 || (d->n_fixed_timesteps > 0 && !d->fixed_timesteps))
    return fail(TB200_ERR_INVALID, "fixed_timesteps is NULL with n_fixed_timesteps > 0");
  if (d->n_fixed_dofs < 0 || (d->n_fixed_dofs > 0 && !d->fixed_dofs))
    return fail(TB200_ERR_INVALID, "fixed_dofs is NULL with n_fixed_dofs > 0");
  if (d->n_obstacles < 0 || (d->n_obstacles > 0 && !d->obstacles))
    return fail(TB200_ERR_INVALID, "obstacles is NULL with n_obstacles > 0");
  if (d->n_cart_targets < 0 || (d->n_cart_targets > 0 && !d->cart_targets))
    return fail(TB200_ERR_INVALID, "cart_targets is NULL with n_cart_targets > 0");

  auto P = new tb200_problem();
  std::unique_ptr<tb200_problem> guard(P);
  P->device = device;
  P->B = B; P->T = T; P->D = D; P->N = N;
  DevProblem& dp = P->dp;
  dp.B = B; dp.T = T; dp.D = D; dp.N = N; dp.HB = 2 * D;
  dp.S = d->robot.n_segments; dp.L = d->robot.n_spheres; dp.O = d->n_obstacles;
  dp.obstacles_per_traj = d->obstacles_per_traj;
  dp.n_cart_targets = d->n_cart_targets;

  // ---- robot ---------------------------------------------------------------------------------------
  std::vector<DevSegment> segs(dp.S);
  std::vector<int> seg_q(dp.S, -1);
  for (int s = 0; s < dp.S; ++s) {
    const tb200_segment& g = d->robot.segments[s];
    if (g.parent >= s) return fail(TB200_ERR_INVALID, "segments must be topologically ordered");
    if (g.joint_type != TB200_JOINT_FIXED && (g.q_index < 0 || g.q_index >= D)) return fail(TB200_ERR_INVALID, "bad q_index");
    segs[s].parent = g.parent; segs[s].joint_type = g.joint_type; segs[s].q_index = g.joint_type == TB200_JOINT_FIXED ? -1 : g.q_index;
    quatToRot(g.origin_wxyz, segs[s].R);
    for (int i = 0; i < 3; ++i) { segs[s].p[i] = g.origin_xyz[i]; segs[s].axis[i] = g.axis[i]; }
    if (g.joint_type != TB200_JOINT_FIXED) P->ex.qtype[g.q_index] = g.joint_type;
  }
  // Fixed segments nobody refers to (no collision sphere, no Cartesian term) are folded into their children:
  // child.origin <- fixed.origin * child.origin.  The kernels then carry fewer frames per waypoint (shared memory of
  // the evaluation kernel: 12 doubles per frame and waypoint).
  std::vector<int> remap(dp.S, -1);
  {
    std::vector<char> used(dp.S, 0);
    for (int s = 0; s < dp.L; ++s) {
      const int g = d->robot.spheres[s].segment;
      if (g < 0 || g >= dp.S) return fail(TB200_ERR_INVALID, "sphere attached to a bad segment");
      used[g] = 1;
    }
    for (int k = 0; k < d->n_terms; ++k)
      if ((d->terms[k].kind == TB200_TERM_CART_POSE || d->terms[k].kind == TB200_TERM_CART_VEL) && d->terms[k].link >= 0 &&
          d->terms[k].link < dp.S)
        used[d->terms[k].link] = 1;
    std::vector<DevSegment> kept;
    std::vector<DevSegment> acc(dp.S);  // transform from the nearest kept ancestor's frame to this (folded) segment
    for (int s = 0; s < dp.S; ++s) {
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
        remap[s] = static_cast<int>(kept.size());
        g.parent = (g.parent >= 0) ? remap[g.parent] : -1;
        kept.push_back(g);
      }
    }
    segs.swap(kept);
    dp.S = static_cast<int>(segs.size());
  }
  std::vector<DevSphere> sph(std::max(dp.L, 1));
  for (int s = 0; s < dp.L; ++s) {
    const tb200_sphere& sp = d->robot.spheres[s];
    sph[s].segment = remap[sp.segment]; sph[s].r = sp.radius;
    for (int i = 0; i < 3; ++i) sph[s].c[i] = sp.center[i];
    unsigned m = 0;
    for (int a = sph[s].segment; a >= 0; a = segs[a].parent)
      if (segs[a].q_index >= 0) m |= 1u << segs[a].q_index;
    P->ex.sphere_jmask[s] = m;
  }

  // ---- hatch terms into cost / constraint objects (constraints: EQ first, then INEQ) ---------------------
  std::vector<DevJointTerm> jts;
  std::vector<DevCartTerm> cts;
  std::vector<DevObj> costs, eqs, ineqs;
  int n_cart_rows = 0, n_coll_cand = 0, max_rows = 0;
  const int cast_cap = tb200inl_cast_rows_per_pair(d);
  P->cast_cap = cast_cap;
  std::vector<std::pair<int, int>> cart_ref, coll_ref, vel_ref;  // (list id: 0 cost 1 eq 2 ineq, index)
  bool has_vel = false, has_cast = false, has_discrete = false;
  // (term, step) that hatched each object of the three lists (tb200_problem_objects)
  std::vector<std::pair<int, int>> cost_src, eq_src, ineq_src;
  auto note = [&](const std::vector<DevObj>& lst, int k, int step) {
    (&lst == &costs ? cost_src : (&lst == &eqs ? eq_src : ineq_src)).push_back({k, step});
  };
  for (int k = 0; k < d->n_terms; ++k) {
    const tb200_term& tm = d->terms[k];
    if (tm.role != TB200_ROLE_COST && tm.role != TB200_ROLE_CNT) return fail(TB200_ERR_INVALID, "term role must be COST or CNT");
    const bool is_cnt = tm.role == TB200_ROLE_CNT;
    DevObj o{};
    o.is_cnt = is_cnt;
    if (tm.kind == TB200_TERM_JOINT_POS || tm.kind == TB200_TERM_JOINT_VEL || tm.kind == TB200_TERM_JOINT_ACC) {
      o.order = tm.kind - TB200_TERM_JOINT_POS;
      o.first = tm.first_step;
      o.n_steps = tm.last_step - tm.first_step + 1 - o.order;
      if (tm.first_step < 0 || tm.last_step >= T) return fail(TB200_ERR_INVALID, "joint term steps outside the trajectory");
      if (o.n_steps <= 0) return fail(TB200_ERR_INVALID, "joint term: trajectory is too short");
      DevJointTerm jt{};
      bool zero_tol = true;
      for (int j = 0; j < D; ++j) {
        jt.coeffs[j] = tm.coeffs[j]; jt.targets[j] = tm.targets[j]; jt.upper[j] = tm.upper_tols[j]; jt.lower[j] = tm.lower_tols[j];
        zero_tol = zero_tol && std::fabs(tm.upper_tols[j]) < 1e-5 && std::fabs(tm.lower_tols[j]) < 1e-5;
      }
      o.term = static_cast<int>(jts.size());
      jts.push_back(jt);
      if (!is_cnt) {
        o.kind = zero_tol ? OBJ_JOINT_EQ_COST : OBJ_JOINT_INEQ_COST;
        o.n_rows = zero_tol ? 0 : 2 * o.n_steps * D;
        costs.push_back(o);
        note(costs, k, tm.first_step);
      } else {
        o.kind = zero_tol ? OBJ_JOINT_EQ_CNT : OBJ_JOINT_INEQ_CNT;
        o.n_rows = (zero_tol ? 1 : 2) * o.n_steps * D;
        (zero_tol ? eqs : ineqs).push_back(o);
        note(zero_tol ? eqs : ineqs, k, tm.first_step);
      }
      max_rows += o.n_rows;
    } else if (tm.kind == TB200_TERM_CART_POSE) {
      if (tm.first_step < 0 || tm.first_step >= T) return fail(TB200_ERR_INVALID, "cart_pose timestep outside the trajectory");
      if (tm.link < 0 || tm.link >= d->robot.n_segments) return fail(TB200_ERR_INVALID, "cart_pose link out of range");
      if (tm.target_slot >= d->n_cart_targets) return fail(TB200_ERR_INVALID, "cart_pose target_slot out of range");
      DevCartTerm ct{};
      quatToRot(tm.source_offset + 3, ct.src_R);
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
      o.term = static_cast<int>(cts.size());
      o.src_off = n_cart_rows;
      o.n_rows = ct.n_idx;
      cts.push_back(ct);
      n_cart_rows += ct.n_idx;
      max_rows += ct.n_idx;
      if (is_cnt) { cart_ref.push_back({1, static_cast<int>(eqs.size())}); eqs.push_back(o); }
      else { cart_ref.push_back({0, static_cast<int>(costs.size())}); costs.push_back(o); }
      note(is_cnt ? eqs : costs, k, tm.first_step);
    } else if (tm.kind == TB200_TERM_COLLISION) {
      if (tm.evaluator_type < TB200_COLL_DISCRETE || tm.evaluator_type > TB200_COLL_LVS_CONTINUOUS)
        return fail(TB200_ERR_INVALID, "unknown collision evaluator type");
      if (dp.L == 0 || dp.O == 0) return fail(TB200_ERR_INVALID, "collision term needs robot spheres and obstacles");
      if (tm.n_fixed_steps < 0 || tm.n_fixed_steps > 8) return fail(TB200_ERR_INVALID, "collision term: n_fixed_steps outside [0, 8]");
      const bool cast = tm.evaluator_type != TB200_COLL_DISCRETE;
      if (cast && tm.evaluator_type != TB200_COLL_CONTINUOUS && !(tm.longest_valid_segment_length > 0.0))
        return fail(TB200_ERR_INVALID, "longest_valid_segment_length must be positive");
      if ((cast && has_discrete) || (!cast && has_cast))
        return fail(TB200_ERR_UNSUPPORTED, "discrete and continuous collision terms in one problem are not supported");
      (cast ? has_cast : has_discrete) = true;
      // discrete: one object per non-fixed step (problem_description.cpp:1762-1775, 1824-1833); continuous: one per
      // step pair [first, last) with the expression type taken from the fixed steps (:1714-1760, 1776-1819)
      for (int t = tm.first_step; cast ? t < tm.last_step : t <= tm.last_step; ++t) {
        bool fixed = false, next_fixed = false;
        for (int f = 0; f < tm.n_fixed_steps; ++f) {
          fixed |= tm.fixed_steps[f] == t;
          next_fixed |= tm.fixed_steps[f] == t + 1;
        }
        if (!cast && fixed) continue;
        if (t < 0 || t + (cast ? 1 : 0) >= T) return fail(TB200_ERR_INVALID, "collision step outside the trajectory");
        DevObj c = o;
        c.kind = cast ? OBJ_COLL_CAST : OBJ_COLL;
        c.first = t;
        c.src_off = n_coll_cand;
        c.n_rows = cast ? cast_cap : dp.L * dp.O;  // continuous: room for cast_cap active contacts of the step pair
        c.coeff = tm.coeff; c.margin = tm.margin; c.buffer = tm.margin_buffer;
        // (two adjacent fixed steps take the START_FIXED_END_FREE branch: the reference's throw is unreachable)
        // bit 2: LVS_DISCRETE = a discrete test at every state of the sub-trajectory instead of a swept one per sub-segment
        c.pad1 = cast ? ((fixed ? 1 : 0) | ((!fixed && next_fixed) ? 2 : 0) | (tm.evaluator_type == TB200_COLL_LVS_DISCRETE ? 4 : 0)) : 0;
        c.lvs = (tm.evaluator_type == TB200_COLL_CONTINUOUS) ? std::numeric_limits<double>::max() : tm.longest_valid_segment_length;
        if (is_cnt) { coll_ref.push_back({2, static_cast<int>(ineqs.size())}); ineqs.push_back(c); }
        else { coll_ref.push_back({0, static_cast<int>(costs.size())}); costs.push_back(c); }
        note(is_cnt ? ineqs : costs, k, t);
      }
    } else if (tm.kind == TB200_TERM_CART_VEL) {
      // CartVelTermInfo::hatch (problem_description.cpp:1011-1057): one object per step pair (t, t+1)
      if (tm.link < 0 || tm.link >= d->robot.n_segments) return fail(TB200_ERR_INVALID, "cart_vel link out of range");
      unsigned lm = 0;
      for (int a = remap[tm.link]; a >= 0; a = segs[a].parent)
        if (segs[a].q_index >= 0) lm |= 1u << segs[a].q_index;
      for (int t = tm.first_step; t <= tm.last_step; ++t) {
        if (t < 0 || t + 1 >= T) return fail(TB200_ERR_INVALID, "cart_vel: step pair beyond the trajectory");
        DevObj c = o;
        c.kind = OBJ_CART_VEL;
        c.first = t;
        c.link = remap[tm.link];
        c.src_off = n_cart_rows;
        c.n_rows = 6;
        c.pad1 = static_cast<int>(lm);
        c.lvs = tm.max_displacement;
        n_cart_rows += 6;
        max_rows += 6;
        has_vel = true;
        if (is_cnt) { vel_ref.push_back({2, static_cast<int>(ineqs.size())}); ineqs.push_back(c); }
        else { vel_ref.push_back({0, static_cast<int>(costs.size())}); costs.push_back(c); }
        note(is_cnt ? ineqs : costs, k, t);
      }
    } else {
      return fail(TB200_ERR_INVALID, "unknown term kind");
    }
  }
  for (auto* lst : {&costs, &ineqs})
    for (DevObj& o : *lst)
      if (o.kind == OBJ_COLL || o.kind == OBJ_COLL_CAST) {
        n_coll_cand += o.n_rows;
        max_rows += o.n_rows;
      }
  P->obj_src = cost_src;
  P->obj_src.insert(P->obj_src.end(), eq_src.begin(), eq_src.end());
  P->obj_src.insert(P->obj_src.end(), ineq_src.begin(), ineq_src.end());
  P->cost_objs = costs;
  P->cnt_objs = eqs;
  P->cnt_objs.insert(P->cnt_objs.end(), ineqs.begin(), ineqs.end());
  const int n_eq = static_cast<int>(eqs.size());
  for (auto& r : cart_ref) {
    DevObj o = (r.first == 0) ? costs[r.second] : eqs[r.second];
    o.pad0 = r.second;
    P->cart_objs.push_back(o);
  }
  for (auto& r : vel_ref) {
    DevObj o = (r.first == 0) ? costs[r.second] : ineqs[r.second];
    o.pad0 = (r.first == 0) ? r.second : n_eq + r.second;
    P->vel_objs.push_back(o);
  }
  // collision objects in the order the QP kernel meets them: cost objects first, then constraint objects
  for (int pass = 0; pass < 2; ++pass)
    for (auto& r : coll_ref) {
      if ((pass == 0) != (r.first == 0)) continue;
      DevObj o = (r.first == 0) ? costs[r.second] : ineqs[r.second];
      o.pad0 = (r.first == 0) ? r.second : n_eq + r.second;
      P->coll_objs.push_back(o);
    }
  // candidates are laid out in P->coll_objs order (src_off) : re-number so that layout == kernel order
  {
    int off = 0, k = 0;
    for (auto& o : P->coll_objs) {
      o.src_off = off;
      o.target_slot = k;  // position in the kernel order: where the evaluation kernel leaves the object's value
      off += o.n_rows;
      DevObj& m = o.is_cnt ? P->cnt_objs[o.pad0] : P->cost_objs[o.pad0];
      m.src_off = o.src_off;
      m.target_slot = k++;
    }
  }
  // fixed rows
  std::vector<int> fixed;
  for (int k = 0; k < d->n_fixed_timesteps; ++k) {
    const int t = d->fixed_timesteps[k];
    if (t < 0 || t >= T) return fail(TB200_ERR_INVALID, "Fixed timestep index is outside the bounds of the initial trajectory.");
    for (int j = 0; j < D; ++j) fixed.push_back(t * D + j);
  }
  for (int k = 0; k < d->n_fixed_dofs; ++k) {
    const int j = d->fixed_dofs[k];
    if (j < 0 || j >= D) return fail(TB200_ERR_INVALID, "DOF(aka Joint) indice is greater than the number of DOF available.");
    for (int t = 0; t < T; ++t) {
      bool skip = false;
      for (int f = 0; f < d->n_fixed_timesteps; ++f) skip |= d->fixed_timesteps[f] == t;
      if (!skip) fixed.push_back(t * D + j);
    }
  }
  max_rows += static_cast<int>(fixed.size());
  max_rows = std::max(max_rows, 1);

  // ---- quadratic objective of the state-independent costs: P = M + M' (osqp_interface.cpp:170-211) ------
  const int W = dp.HB + 1;
  std::vector<double> Pband(static_cast<size_t>(N) * W, 0.0), qlin(N, 0.0);
  for (const DevObj& o : costs) {
    if (o.kind != OBJ_JOINT_EQ_COST) continue;
    static const double wst[3][3] = {{1, 0, 0}, {-1, 1, 0}, {1, -2, 1}};
    const DevJointTerm& jt = jts[o.term];
    for (int t = o.first; t < o.first + o.n_steps; ++t)
      for (int j = 0; j < D; ++j)
        for (int a = 0; a <= o.order; ++a) {
          const int ia = (t + a) * D + j;
          qlin[ia] += -2.0 * jt.coeffs[j] * jt.targets[j] * wst[o.order][a];
          for (int bb = 0; bb <= a; ++bb) {
            const int ib = (t + bb) * D + j;
            Pband[static_cast<size_t>(ia) * W + (ia - ib)] += 2.0 * jt.coeffs[j] * wst[o.order][a] * wst[o.order][bb];
          }
        }
  }

  {  // the structurally non-zero offsets of the band (the kernels visit only these)
    dp.n_band = 0;
    for (int k = 0; k < W; ++k) {
      bool nz = false;
      for (int i = k; i < N && !nz; ++i) nz = Pband[static_cast<size_t>(i) * W + k] != 0.0;
      if (nz) dp.band_offs[dp.n_band++] = k;
    }
  }
  // ---- layout ---------------------------------------------------------------------------------------
  dp.n_costs = static_cast<int>(P->cost_objs.size());
  dp.n_cnts = static_cast<int>(P->cnt_objs.size());
  dp.n_cart_rows = n_cart_rows;
  const int CN = (has_vel || has_cast) ? std::max(2 * D, 3) : std::max(D, 3);  // coefficients per (padded) QP row
  dp.cart_stride = has_vel ? 2 * D : D;
  dp.n_coll_cand = n_coll_cand;
  dp.coll_stride = has_cast ? 2 * D + 3 : D + 3;
  dp.n_fixed = static_cast<int>(fixed.size());
  dp.max_rows = max_rows;
  dp.row_stride = qp_row_stride(CN);
  dp.coll_words = std::max(1, ((has_cast ? cast_cap : dp.L * dp.O) + 63) / 64);
  dp.n_coll_objs = static_cast<int>(P->coll_objs.size());
  P->ex.n_cart_objs = static_cast<int>(P->cart_objs.size());
  P->ex.n_coll_objs = dp.n_coll_objs;
  P->ex.n_vel_objs = static_cast<int>(P->vel_objs.size());
  P->ex.cast = has_cast ? 1 : 0;
  P->ex.cast_cap = cast_cap;
  for (int sg = 0; sg < dp.S; ++sg)
    if (segs[sg].q_index >= 0) P->ex.joint_seg[segs[sg].q_index] = sg;
  P->ex.n_joint_objs = 0;
  {
    int idx = 0;
    auto note = [&](const DevObj& o) {
      if (o.kind <= OBJ_JOINT_INEQ_CNT) {
        if (P->ex.n_joint_objs < 8) P->ex.joint_obj_idx[P->ex.n_joint_objs] = idx;
        P->ex.n_joint_objs++;
      }
      ++idx;
    };
    for (const DevObj& o : P->cost_objs) note(o);
    for (const DevObj& o : P->cnt_objs) note(o);
    if (P->ex.n_joint_objs > 8) return fail(TB200_ERR_UNSUPPORTED, "more than 8 joint-space cost/constraint objects");
    if (dp.O > 64) return fail(TB200_ERR_UNSUPPORTED, "more than 64 obstacle spheres per trajectory");
  }
  P->layout.n_costs = dp.n_costs;
  P->layout.n_cnts = dp.n_cnts;
  P->layout.n_cart_rows = n_cart_rows;
  P->layout.cart_jac_stride = dp.cart_stride;
  P->layout.n_coll_cand = n_coll_cand;
  P->layout.coll_row_stride = dp.coll_stride;
  P->layout.n_vars = N;

  // ---- kernel resources --------------------------------------------------------------------------------
  const EvalSmem es = eval_smem_layout(T, D, dp.L, dp.n_coll_objs, dp.n_coll_objs * dp.coll_words, dp.S, P->ex.n_joint_objs,
                                       P->ex.n_vel_objs, P->ex.cast, cast_cap, dp.n_costs + dp.n_cnts);
  P->pair_rows = (CN > std::max(D, 3));
  P->eval_smem = static_cast<size_t>(es.total) * sizeof(double);
  const bool factor_global = D > 8;  // = FG of qp_step: blocks of 2*D > 16 never fit
  const QpSmem qs = qp_smem_layout(N, 2 * D, dp.row_stride, CN, max_rows, factor_global);
  const int Np = qp_block_count(N, 2 * D) * 2 * D;
  dp.list_stride = static_cast<size_t>(Np + 1) + static_cast<size_t>(max_rows) * CN + dp.n_costs + dp.n_cnts + 2;
  P->qp_smem = static_cast<size_t>(qs.total) * sizeof(double);
  if (P->eval_smem > 226 * 1024 || P->qp_smem > 226 * 1024)
    return fail(TB200_ERR_UNSUPPORTED, "problem does not fit the 227 KB shared memory of one CTA");
  if (CN > 32) return fail(TB200_ERR_UNSUPPORTED, "more than 32 coefficients per QP row");
  if (!solve_kernel_for(D, P->pair_rows) || !eval_kernel_for(D))
    return fail(TB200_ERR_UNSUPPORTED, P->pair_rows ? "no kernel instance with two-waypoint rows (CartVel, continuous collision) for this number of joints"
                                                    : "no kernel instance for this number of joints");
  // ---- from here on the device is needed ---------------------------------------------------------------------
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(TB200_ERR_NO_DEVICE, "no CUDA device: trajopt_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(TB200_ERR_INVALID, "bad device ordinal");
  CK(cudaSetDevice(device));
  {  // the QP step calls its hot functions through pointers (standard calling convention): make sure the per-thread stack
     // covers the deepest chain (ptxas reports < 3 KB for the chains it can follow)
    size_t cur = 0;
    CK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
    if (cur < 6144) CK(cudaDeviceSetLimit(cudaLimitStackSize, 6144));
  }
  CK(cudaFuncSetAttribute(eval_kernel_for(D), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P->eval_smem)));
  P->solve_smem = std::max(P->qp_smem, P->eval_smem);  // the QP step and the evaluation step share one buffer
  CK(cudaFuncSetAttribute(solve_kernel_for(D, P->pair_rows), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P->solve_smem)));
  {
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    P->n_sm = std::max(1, sms);
  }
  if (const char* e = std::getenv("TB200_QUANTUM")) P->quantum = std::max(1, std::atoi(e));
  // TB200_GENERIC_QP_PASSES=1: termination checks and polish refinement by the generic passes of the QP solver instead
  // of the check fused into the ADMM block and polish_passes (same decisions; the switch exists to compare the two)
  {
    const char* e = std::getenv("TB200_GENERIC_QP_PASSES");
    P->dp.qp_fast_passes = (e && std::atoi(e) != 0) ? 0 : 1;
  }
  CK(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking));

  // ---- device buffers ------------------------------------------------------------------------------------
#define ALLOC(buf, count) CK(P->buf.alloc(count))
#define UPLOAD(buf, vec) \
  CK(P->buf.alloc((vec).size())); \
  if (!(vec).empty()) CK(cudaMemcpy(P->buf.p, (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice))
  UPLOAD(segs, segs);
  UPLOAD(spheres, sph);
  std::vector<double> lo(d->robot.lower, d->robot.lower + D), up(d->robot.upper, d->robot.upper + D);
  UPLOAD(lower, lo);
  UPLOAD(upper, up);
  UPLOAD(Pband, Pband);
  UPLOAD(qlin, qlin);
  UPLOAD(d_cost_objs, P->cost_objs);
  UPLOAD(d_cnt_objs, P->cnt_objs);
  UPLOAD(d_cart_objs, P->cart_objs);
  UPLOAD(d_coll_objs, P->coll_objs);
  UPLOAD(d_vel_objs, P->vel_objs);
  UPLOAD(joint_terms, jts);
  UPLOAD(cart_terms, cts);
  UPLOAD(fixed_vars, fixed);
  const size_t Bs = B;
  ALLOC(init_traj, Bs * N);
  ALLOC(cart_targets, Bs * std::max(1, d->n_cart_targets) * 7);
  ALLOC(obstacles, (d->obstacles_per_traj ? Bs : 1) * std::max(1, dp.O) * 4);
  ALLOC(x, Bs * N); ALLOC(new_x, Bs * N); ALLOC(trust, Bs); ALLOC(merit_coeffs, Bs * std::max(1, dp.n_cnts));
  ALLOC(cost_vals, Bs * std::max(1, dp.n_costs)); ALLOC(cnt_viols, Bs * std::max(1, dp.n_cnts));
  ALLOC(new_cost_vals, Bs * std::max(1, dp.n_costs)); ALLOC(new_cnt_viols, Bs * std::max(1, dp.n_cnts));
  ALLOC(model_cost_vals, Bs * std::max(1, dp.n_costs)); ALLOC(model_cnt_viols, Bs * std::max(1, dp.n_cnts));
  ALLOC(cart_err, 2 * Bs * std::max(1, n_cart_rows)); ALLOC(cart_jac, 2 * Bs * std::max(1, n_cart_rows) * dp.cart_stride);
  ALLOC(coll_rows, 2 * Bs * std::max(1, n_coll_cand) * dp.coll_stride);
  ALLOC(coll_mask, 2 * Bs * std::max(1, dp.n_coll_objs * dp.coll_words));
  ALLOC(rows, Bs * max_rows * dp.row_stride); ALLOC(row_ints, Bs * max_rows * RI_NINTS);
  ALLOC(lists, Bs * dp.list_stride);
  ALLOC(ws_x, Bs * N); ALLOC(ws_yb, Bs * N); ALLOC(scratch, Bs * 5 * Np); ALLOC(qp_done, Bs); ALLOC(ws_rho, Bs); ALLOC(ws_meta, Bs * 8);
  ALLOC(lvs_overflow, Bs);
  ALLOC(work_counter, 1);
  {
    int per_sm = 1;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, eval_kernel_for(D), kEvalThreads, P->eval_smem));
    P->eval_grid = std::max(1, std::min(B, std::max(1, per_sm) * P->n_sm));
  }
  // contact lists of the continuous collision evaluator: one per resident warp of the largest launch (4 doubles a contact)
  ALLOC(cast_scratch, has_cast ? static_cast<size_t>(std::max(P->eval_grid, std::min(B, P->n_sm))) * (kEvalThreads / 32) * 4 * cast_cap : 0);
  // per-CTA regions (the persistent kernel and the kernel-level QP entry point both launch at most one CTA per SM):
  // a factor that does not fit shared memory, and the column-major copy of rows that do not
  P->factor_grid = static_cast<size_t>(P->n_sm);  // per resident CTA: the factor of wide blocks, or the rows of the partition inverses
  ALLOC(factor_g, P->factor_grid * qp_cta_global_doubles(N, 2 * D));
  dp.soa_stride = (max_rows > qs.row_cap) ? qp_soa_doubles(max_rows, CN) : 0;
  ALLOC(soa, static_cast<size_t>(P->n_sm) * dp.soa_stride);
  {
    std::vector<int> chain(static_cast<size_t>(dp.S) * (kMaxSeg + 1), 0);
    for (int sg = 0; sg < dp.S; ++sg) {
      std::vector<int> up;
      for (int a = sg; a >= 0; a = segs[a].parent) up.push_back(a);
      int* c = chain.data() + static_cast<size_t>(sg) * (kMaxSeg + 1);
      c[0] = static_cast<int>(up.size());
      for (size_t k = 0; k < up.size(); ++k) c[1 + k] = up[up.size() - 1 - k];
    }
    UPLOAD(link_chain, chain);
  }
  ALLOC(status, Bs); ALLOC(sqp_iter, Bs); ALLOC(merit_round, Bs); ALLOC(qp_failures, Bs); ALLOC(qp_status, Bs);
  ALLOC(cur_buf, Bs); ALLOC(n_qp_solves, Bs); ALLOC(n_func_evals, Bs); ALLOC(n_admm_iters, Bs); ALLOC(active_count, 2);
  ALLOC(dbg, Bs * 16);
  ALLOC(sched_state, Bs); ALLOC(sched_timers, 8 + 2 * Bs);
  ALLOC(clock_start, 1); ALLOC(sqp_top, Bs); ALLOC(ended_by, Bs); ALLOC(group_done, Bs);
  ALLOC(g_best, Bs); ALLOC(g_status, Bs); ALLOC(g_n_converged, Bs); ALLOC(g_total_cost, Bs); ALLOC(g_x, Bs * N);
  ALLOC(trace_len, Bs);
  ALLOC(x_tmp, Bs * N); ALLOC(trust_tmp, Bs); ALLOC(tmp_iters, Bs); ALLOC(tmp_polish, Bs);
#undef ALLOC
#undef UPLOAD
  dp.segs = P->segs.p; dp.spheres = P->spheres.p; dp.lower = P->lower.p; dp.upper = P->upper.p;
  dp.cost_objs = P->d_cost_objs.p; dp.cnt_objs = P->d_cnt_objs.p; dp.joint_terms = P->joint_terms.p;
  dp.cart_terms = P->cart_terms.p; dp.fixed_vars = P->fixed_vars.p; dp.Pband = P->Pband.p; dp.qlin = P->qlin.p;
  dp.init_traj = P->init_traj.p; dp.cart_targets = P->cart_targets.p; dp.obstacles = P->obstacles.p;
  dp.x = P->x.p; dp.new_x = P->new_x.p; dp.trust = P->trust.p; dp.merit_coeffs = P->merit_coeffs.p;
  dp.cost_vals = P->cost_vals.p; dp.cnt_viols = P->cnt_viols.p; dp.new_cost_vals = P->new_cost_vals.p;
  dp.new_cnt_viols = P->new_cnt_viols.p; dp.model_cost_vals = P->model_cost_vals.p; dp.model_cnt_viols = P->model_cnt_viols.p;
  dp.status = P->status.p; dp.sqp_iter = P->sqp_iter.p; dp.merit_round = P->merit_round.p; dp.qp_failures = P->qp_failures.p;
  dp.qp_status = P->qp_status.p; dp.cur_buf = P->cur_buf.p; dp.n_qp_solves = P->n_qp_solves.p;
  dp.n_func_evals = P->n_func_evals.p; dp.n_admm_iters = P->n_admm_iters.p; dp.active_count = P->active_count.p;
  dp.cart_err = P->cart_err.p; dp.cart_jac = P->cart_jac.p; dp.coll_rows = P->coll_rows.p; dp.coll_mask = P->coll_mask.p;
  dp.rows = P->rows.p; dp.row_ints = P->row_ints.p; dp.lists = P->lists.p; dp.ws_x = P->ws_x.p; dp.ws_yb = P->ws_yb.p;
  dp.scratch = P->scratch.p; dp.ws_meta = P->ws_meta.p; dp.ws_rho = P->ws_rho.p; dp.dbg = P->dbg.p; dp.sched_state = P->sched_state.p; dp.sched_timers = P->sched_timers.p; dp.trace_len = P->trace_len.p; dp.trace = nullptr; dp.trace_cap = 0;
  dp.soa = P->soa.p;
  dp.clock_start = P->clock_start.p; dp.sqp_top = P->sqp_top.p; dp.ended_by = P->ended_by.p; dp.group_done = P->group_done.p;
  dp.factor_g = P->factor_g.p; dp.lvs_overflow = P->lvs_overflow.p; dp.qp_done = P->qp_done.p;
  P->ex.link_chain = P->link_chain.p;
  P->ex.work_counter = P->work_counter.p;
  P->ex.cast_scratch = P->cast_scratch.p;
  P->ex.cart_objs = P->d_cart_objs.p;
  P->ex.coll_objs = P->d_coll_objs.p;
  P->ex.vel_objs = P->d_vel_objs.p;
  // settings
  const tb200_qp_settings& q = d->qp;
  dp.qp = QpSettings{q.rho, q.sigma, q.alpha, q.eps_abs, q.eps_rel, q.eps_prim_inf, q.eps_dual_inf, q.delta,
                     q.adaptive_rho_tolerance, q.max_iter, q.scaling, q.check_termination, q.adaptive_rho,
                     q.adaptive_rho_interval, q.polishing, q.polish_refine_iter, q.warm_starting,
                     q.early_polish_every, q.early_polish_from};
  const tb200_sqp_params& s = d->sqp;
  dp.sqp = SqpParams{s.improve_ratio_threshold, s.min_trust_box_size, s.min_approx_improve, s.min_approx_improve_frac,
                     s.trust_shrink_ratio, s.trust_expand_ratio, s.cnt_tolerance, s.max_merit_coeff_increases,
                     s.merit_coeff_increase_ratio, s.initial_merit_error_coeff, s.trust_box_size, s.max_iter,
                     s.max_qp_solver_failures, s.inflate_constraints_individually, 0, s.max_time};
  setGroups(dp, d->group_size, d->group_stop);
  int rc = tb200_problem_set_inputs(P, d->init_traj, d->cart_targets, d->obstacles);
  if (rc != TB200_OK) return rc;
  *out = guard.release();
  return TB200_OK;
}

void tb200_problem_destroy(tb200_problem* p) { delete p; }

int tb200_problem_layout(const tb200_problem* p, tb200_layout* out) {
  if (!p || !out) return fail(TB200_ERR_INVALID, "null argument");
  *out = p->layout;
  return TB200_OK;
}

int tb200_problem_set_sqp_params(tb200_problem* P, const tb200_sqp_params* s) {
  if (!P || !s) return fail(TB200_ERR_INVALID, "null argument");
  P->dp.sqp = SqpParams{s->improve_ratio_threshold, s->min_trust_box_size, s->min_approx_improve, s->min_approx_improve_frac,
                        s->trust_shrink_ratio, s->trust_expand_ratio, s->cnt_tolerance, s->max_merit_coeff_increases,
                        s->merit_coeff_increase_ratio, s->initial_merit_error_coeff, s->trust_box_size, s->max_iter,
                        s->max_qp_solver_failures, s->inflate_constraints_individually, 0, s->max_time};
  return TB200_OK;
}

int tb200_problem_set_groups(tb200_problem* P, int32_t group_size, int32_t group_stop) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  if (int rc = checkGroups(P->B, group_size, group_stop)) return rc;
  setGroups(P->dp, group_size, group_stop);
  return TB200_OK;
}

int tb200_problem_set_inputs(tb200_problem* P, const double* init_traj, const double* cart_targets, const double* obstacles) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  CK(cudaSetDevice(P->device));
  P->timing.h2d_bytes = 0;
  if (init_traj) {
    CK(cudaMemcpyAsync(P->init_traj.p, init_traj, P->init_traj.n * sizeof(double), cudaMemcpyHostToDevice, P->stream));
    P->timing.h2d_bytes += static_cast<int64_t>(P->init_traj.n * sizeof(double));
  }
  if (cart_targets && P->dp.n_cart_targets > 0) {
    CK(cudaMemcpyAsync(P->cart_targets.p, cart_targets, P->cart_targets.n * sizeof(double), cudaMemcpyHostToDevice, P->stream));
    P->timing.h2d_bytes += static_cast<int64_t>(P->cart_targets.n * sizeof(double));
  }
  if (obstacles && P->dp.O > 0) {
    CK(cudaMemcpyAsync(P->obstacles.p, obstacles, P->obstacles.n * sizeof(double), cudaMemcpyHostToDevice, P->stream));
    P->timing.h2d_bytes += static_cast<int64_t>(P->obstacles.n * sizeof(double));
  }
  CK(cudaStreamSynchronize(P->stream));
  return TB200_OK;
}

namespace {
__global__ void reset_state_kernel(DevProblem p, int* log_len, int* log_dropped) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) {
    p.active_count[0] = p.B;
    p.active_count[1] = 0;
    for (int k = 0; k < 8; ++k) p.sched_timers[k] = (k == 4) ? ~0ull : 0ull;
    *p.clock_start = global_ns();  // the time limit's clock: one start for the whole batch (DESIGN.md section 6)
  }
  if (b >= p.B) return;
  p.status[b] = 5;
  p.sqp_iter[b] = 1;
  p.merit_round[b] = 0;
  p.qp_failures[b] = 0;
  p.qp_status[b] = 0;
  p.cur_buf[b] = 0;
  p.n_qp_solves[b] = 0;
  p.n_func_evals[b] = 0;
  p.n_admm_iters[b] = 0;
  p.trust[b] = p.sqp.trust_box_size;
  for (int c = 0; c < p.n_cnts; ++c) p.merit_coeffs[static_cast<size_t>(b) * p.n_cnts + c] = p.sqp.initial_merit_error_coeff;
  for (int k = 0; k < 8; ++k) p.ws_meta[b * 8 + k] = 0;
  p.qp_done[b] = 0;
  p.lvs_overflow[b] = 0;
  p.sched_state[b] = 0;
  p.sched_timers[8 + b] = 0ull;
  p.sched_timers[8 + p.B + b] = 0ull;
  p.ws_rho[b] = p.qp.rho;
  p.trace_len[b] = 0;
  p.sqp_top[b] = 0;  // (set by the initial evaluation)
  p.ended_by[b] = 0;
  if (b < p.B / p.group_size) p.group_done[b] = 0;
  if (log_len) {  // (the SQP log is on)
    log_len[b] = 0;
    log_dropped[b] = 0;
  }
}

struct GroupOut {
  int *best, *status, *n_converged;
  double *total_cost, *x;
};
// Selection key of one seed (tb200_group_results): not converged, its worst constraint violation when not converged, total
// cost, index; a NaN reads as +inf.  Smaller is better.
struct SeedKey {
  int failed;
  double viol, cost;
  int index;
};
__device__ __forceinline__ bool key_less(const SeedKey& a, const SeedKey& b) {
  if (a.failed != b.failed) return a.failed < b.failed;
  if (a.viol != b.viol) return a.viol < b.viol;
  if (a.cost != b.cost) return a.cost < b.cost;
  return a.index < b.index;
}
__device__ __forceinline__ double nan_as_inf(double v) { return v != v ? CUDART_INF : v; }
// total_cost as tb200_fetch_results sums it (results_.total_cost = vecSum(cost_vals)): the same bits
__device__ __forceinline__ double total_cost_of(const DevProblem& p, int b) {
  double s = 0;
  for (int i = 0; i < p.n_costs; ++i) s += p.cost_vals[static_cast<size_t>(b) * p.n_costs + i];
  return s;
}

// The best seed of every group from the final per-trajectory results: one warp per group, each lane keys the seeds
// lane, lane + 32, ... of its group, a butterfly reduction leaves the minimum on every lane, and the warp copies the
// winner's x (two doubles per load when the rows are 16-byte aligned).
__global__ void group_select_kernel(const DevProblem p, const GroupOut g) {
  const int lane = threadIdx.x & 31;
  const int grp = static_cast<int>((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int G = p.group_size;
  if (grp >= p.B / G) return;  // (whole warps)
  SeedKey best{2, CUDART_INF, CUDART_INF, INT_MAX};
  int n_conv = 0;
  for (int k = lane; k < G; k += 32) {
    const int b = grp * G + k;
    SeedKey s{p.status[b] != 0, 0.0, nan_as_inf(total_cost_of(p, b)), b};
    if (s.failed) {
      const double* kv = p.cnt_viols + static_cast<size_t>(b) * p.n_cnts;
      for (int i = 0; i < p.n_cnts; ++i) s.viol = fmax(s.viol, nan_as_inf(kv[i]));
    }
    n_conv += !s.failed;
    if (key_less(s, best)) best = s;
  }
  for (int o = 16; o > 0; o >>= 1) {
    SeedKey other;
    other.failed = __shfl_xor_sync(0xffffffffu, best.failed, o);
    other.viol = __shfl_xor_sync(0xffffffffu, best.viol, o);
    other.cost = __shfl_xor_sync(0xffffffffu, best.cost, o);
    other.index = __shfl_xor_sync(0xffffffffu, best.index, o);
    if (key_less(other, best)) best = other;
    n_conv += __shfl_xor_sync(0xffffffffu, n_conv, o);
  }
  const int w = best.index;
  if (lane == 0) {
    g.best[grp] = w;
    g.status[grp] = p.status[w];
    g.total_cost[grp] = total_cost_of(p, w);
    g.n_converged[grp] = n_conv;
  }
  const double* src = p.x + static_cast<size_t>(w) * p.N;
  double* dst = g.x + static_cast<size_t>(grp) * p.N;
  if ((p.N & 1) == 0) {
    const double2* s2 = reinterpret_cast<const double2*>(src);
    double2* d2 = reinterpret_cast<double2*>(dst);
    for (int i = lane; i < p.N / 2; i += 32) d2[i] = s2[i];
  } else {
    for (int i = lane; i < p.N; i += 32) dst[i] = src[i];
  }
}

// Launches the selection for groups of G seeds on the solver's stream.
int launchGroupSelect(tb200_problem* P, int G) {
  DevProblem dp = P->dp;
  dp.group_size = G;
  const int NG = dp.B / G;
  const GroupOut g{P->g_best.p, P->g_status.p, P->g_n_converged.p, P->g_total_cost.p, P->g_x.p};
  group_select_kernel<<<(NG + 3) / 4, 128, 0, P->stream>>>(dp, g);
  CK(cudaGetLastError());
  P->selected = true;
  return TB200_OK;
}

// Doubles of one SQP log record (DevProblem::log): header, merit coefficients, model values, exact values, point.
size_t logStride(const tb200_problem* P, int with_x) {
  const size_t nc = P->dp.n_costs, nk = P->dp.n_cnts;
  return kLogHeader + 3 * nk + 2 * nc + (with_x ? static_cast<size_t>(P->N) : 0);
}
// The log setting of tb200_problem_set_sqp_log takes effect here, at the start of a solve: the record buffer is
// (re)allocated when its shape changed and released when the log is off.
int applyLogSetting(tb200_problem* P) {
  EvalExtra& ex = P->ex;
  const int cap = P->log_cap_next, wx = P->log_with_x_next;
  const size_t stride = logStride(P, wx);
  const bool keep = cap > 0 && ex.log != nullptr && ex.log_cap == cap && ex.log_with_x == wx;
  // off until the buffers of the new setting exist: a failed allocation leaves the log off, not pointing at freed memory
  P->log_solved = false;
  ex.log = nullptr; ex.log_len = ex.log_dropped = nullptr;
  ex.log_cap = ex.log_stride = ex.log_with_x = 0;
  if (!keep) {
    P->log.release(); P->log_len.release(); P->log_dropped.release();
    if (cap == 0) return TB200_OK;
    cudaError_t e = P->log.alloc(static_cast<size_t>(P->B) * cap * stride);
    if (e == cudaSuccess) e = P->log_len.alloc(P->B);
    if (e == cudaSuccess) e = P->log_dropped.alloc(P->B);
    if (e != cudaSuccess) {
      P->log.release(); P->log_len.release(); P->log_dropped.release();
      return fail(TB200_ERR_CUDA, std::string("SQP log buffer of ") + std::to_string(cap) + " records: " + cudaGetErrorString(e));
    }
  }
  ex.log = P->log.p; ex.log_len = P->log_len.p; ex.log_dropped = P->log_dropped.p;
  ex.log_cap = cap; ex.log_stride = static_cast<int>(stride); ex.log_with_x = wx;
  P->log_solved = true;
  return TB200_OK;
}

cudaEvent_t getEvent(tb200_problem* P, size_t i) {
  while (P->events.size() <= i) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    P->events.push_back(e);
  }
  return P->events[i];
}
}  // namespace

int tb200_solve_batch_resident(tb200_problem* P) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  CK(cudaSetDevice(P->device));
  const DevProblem& dp = P->dp;
  cudaStream_t st = P->stream;
  tb200_timing& tm = P->timing;
  const int64_t h2d = tm.h2d_bytes;
  tm = tb200_timing{};
  tm.h2d_bytes = h2d;
  if (int rc = applyLogSetting(P)) return rc;
  cudaEvent_t e_begin = getEvent(P, 0), e_end = getEvent(P, 1), e_init0 = getEvent(P, 2), e_init1 = getEvent(P, 3);
  CK(cudaEventRecord(e_begin, st));
  reset_state_kernel<<<(dp.B + 127) / 128, 128, 0, st>>>(dp, P->ex.log_len, P->ex.log_dropped);
  if (dp.qp_paths) CK(cudaMemsetAsync(dp.qp_paths, 0, dp.B * sizeof(int), st));
  // the initial evaluation + convexification of every trajectory: one CTA per trajectory (optimizers.cpp:761-783)
  CK(cudaEventRecord(e_init0, st));
  CK(cudaMemsetAsync(P->work_counter.p, 0, sizeof(int), st));
  eval_kernel_for(P->D)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_INIT, nullptr);
  CK(cudaEventRecord(e_init1, st));
  // everything else: one persistent CTA per SM (solve_kernel.cuh); no host round trips until every trajectory is done
  SolveCtl ctl{};
  ctl.mode = SOLVE_FULL;
  ctl.quantum = P->quantum;
  ctl.sched_state = dp.sched_state;
  ctl.timers = dp.sched_timers;
  solve_kernel_for(P->D, P->pair_rows)<<<std::min(dp.B, P->n_sm), kQpThreads, P->solve_smem, st>>>(dp, P->ex, ctl);
  // the best seed of every group, inside the timed region (without groups the identity selection is made only when
  // tb200_fetch_group_results asks for it)
  P->solved_group_size = dp.group_size;
  P->selected = false;
  if (dp.group_size > 1) {
    if (int rc = launchGroupSelect(P, dp.group_size)) return rc;
  }
  CK(cudaEventRecord(e_end, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  float ms = 0, ms_init = 0;
  CK(cudaEventElapsedTime(&ms, e_begin, e_end));
  CK(cudaEventElapsedTime(&ms_init, e_init0, e_init1));
  tm.total_ms = ms;
  unsigned long long tmr[4] = {0, 0, 0, 0};
  CK(cudaMemcpy(tmr, dp.sched_timers, sizeof(tmr), cudaMemcpyDeviceToHost));
  // share of the persistent launch spent in evaluation steps vs QP steps (SM-time, %globaltimer around each step)
  const double in_steps = static_cast<double>(tmr[0]) + static_cast<double>(tmr[1]);
  const double ev_share = in_steps > 0 ? static_cast<double>(tmr[1]) / in_steps : 0.0;
  tm.convexify_ms = ms_init + (ms - ms_init) * ev_share;
  tm.qp_ms = (ms - ms_init) * (1.0 - ev_share);
  tm.convexify_launches = 1 + static_cast<int32_t>(tmr[2]);  // INIT launch + evaluation steps inside the solve
  tm.qp_launches = static_cast<int32_t>(tmr[2]);             // QP steps (one per evaluation step)
  tm.outer_steps = static_cast<int32_t>(tmr[3]);             // trajectory claims of the scheduler
  int active = 0;
  CK(cudaMemcpy(&active, dp.active_count, sizeof(int), cudaMemcpyDeviceToHost));
  // algorithmic HBM bytes of one convexify launch (SURVEY.md §8d): read x, write cart rows, dense collision
  // rows and the exact values, per trajectory
  const int64_t per_traj = 8LL * (dp.N + static_cast<int64_t>(dp.n_coll_cand) * dp.coll_stride +
                                  static_cast<int64_t>(dp.n_cart_rows) * (dp.cart_stride + 1) + dp.n_costs + dp.n_cnts);
  int counters[2] = {0, 0};
  CK(cudaMemcpy(counters, dp.active_count, sizeof(counters), cudaMemcpyDeviceToHost));
  tm.convexify_bytes = per_traj * counters[1];  // summed over all launches: trajectories actually convexified
  if (active > 0) return fail(TB200_ERR_CUDA, "the SQP kernel returned with trajectories still active");
  return TB200_OK;
}

namespace {
// trajectories whose step pairs outgrew the LVS candidate layout (they ended OPT_FAILED; never truncated silently)
int lvsOverflowCount(tb200_problem* P, int* count) {
  *count = 0;
  if (!P->ex.cast) return TB200_OK;
  std::vector<int> f(P->dp.B);
  CK(cudaMemcpy(f.data(), P->lvs_overflow.p, f.size() * sizeof(int), cudaMemcpyDeviceToHost));
  for (int v : f) *count += v != 0;
  return TB200_OK;
}
int lvsOverflowError(tb200_problem* P) {
  int n = 0;
  int rc = lvsOverflowCount(P, &n);
  if (rc != TB200_OK) return rc;
  if (n > 0)
    return fail(TB200_ERR_UNSUPPORTED, std::to_string(n) + " trajectories have a step pair with more than " +
                                           std::to_string(P->cast_cap) + " active continuous-collision contacts (the row block of a pair, "
                                           "tb200inl_cast_rows_per_pair) or more than 32767 longest-valid-segment sub-segments; they are "
                                           "reported OPT_FAILED");
  return TB200_OK;
}
}  // namespace

int tb200_fetch_results(tb200_problem* P, tb200_results* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  const DevProblem& dp = P->dp;
  const size_t B = dp.B;
  int64_t bytes = 0;
  auto pull = [&](void* dst, const void* src, size_t n) {
    if (!dst || n == 0) return cudaSuccess;
    bytes += static_cast<int64_t>(n);
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, P->stream);
  };
  CK(pull(out->x, dp.x, B * dp.N * sizeof(double)));
  CK(pull(out->status, dp.status, B * sizeof(int)));
  CK(pull(out->cost_vals, dp.cost_vals, B * dp.n_costs * sizeof(double)));
  CK(pull(out->cnt_viols, dp.cnt_viols, B * dp.n_cnts * sizeof(double)));
  CK(pull(out->n_qp_solves, dp.n_qp_solves, B * sizeof(int)));
  CK(pull(out->n_func_evals, dp.n_func_evals, B * sizeof(int)));
  CK(pull(out->n_admm_iters, dp.n_admm_iters, B * sizeof(int)));
  std::vector<double> cv;
  if (out->total_cost) {
    cv.resize(B * std::max(1, dp.n_costs));
    CK(cudaMemcpyAsync(cv.data(), dp.cost_vals, B * dp.n_costs * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
  }
  CK(cudaStreamSynchronize(P->stream));
  if (out->total_cost)
    for (size_t b = 0; b < B; ++b) {
      double s = 0;
      for (int i = 0; i < dp.n_costs; ++i) s += cv[b * dp.n_costs + i];  // results_.total_cost = vecSum(cost_vals)
      out->total_cost[b] = s;
    }
  P->timing.d2h_bytes = bytes;
  return TB200_OK;
}

int tb200_fetch_group_results(tb200_problem* P, tb200_group_results* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  if (P->solved_group_size == 0) return fail(TB200_ERR_INVALID, "no solve yet");
  CK(cudaSetDevice(P->device));
  if (!P->selected) {
    if (int rc = launchGroupSelect(P, P->solved_group_size)) return rc;
  }
  const size_t B = P->dp.B, NG = B / P->solved_group_size, N = P->dp.N;
  auto pull = [&](void* dst, const void* src, size_t n) {
    return dst ? cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, P->stream) : cudaSuccess;
  };
  CK(pull(out->best, P->g_best.p, NG * sizeof(int)));
  CK(pull(out->status, P->g_status.p, NG * sizeof(int)));
  CK(pull(out->total_cost, P->g_total_cost.p, NG * sizeof(double)));
  CK(pull(out->x, P->g_x.p, NG * N * sizeof(double)));
  CK(pull(out->n_converged, P->g_n_converged.p, NG * sizeof(int)));
  CK(pull(out->ended_by, P->ended_by.p, B * sizeof(int)));
  CK(cudaStreamSynchronize(P->stream));
  return TB200_OK;
}

int tb200_solve_batch(tb200_problem* P, tb200_results* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  int rc = tb200_solve_batch_resident(P);
  if (rc != TB200_OK) return rc;
  rc = tb200_fetch_results(P, out);
  if (rc != TB200_OK) return rc;
  return lvsOverflowError(P);  // (after the results: the other trajectories of the batch are valid)
}

int tb200_convexify_batch(tb200_problem* P, const double* x, tb200_convexify_out* out) {
  if (!P || !x || !out) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  const DevProblem& dp = P->dp;
  const size_t B = dp.B;
  cudaStream_t st = P->stream;
  CK(cudaMemcpyAsync(P->x_tmp.p, x, B * dp.N * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(P->lvs_overflow.p, 0, B * sizeof(int), st));
  if (P->ex.cast)  // the continuous evaluator writes only its active rows: the rest of the (returned) block reads as zeros
    CK(cudaMemsetAsync(P->coll_rows.p, 0, B * dp.n_coll_cand * dp.coll_stride * sizeof(double), st));
  CK(cudaMemsetAsync(P->work_counter.p, 0, sizeof(int), st));
  cudaEvent_t e0 = getEvent(P, 0), e1 = getEvent(P, 1);
  CK(cudaEventRecord(e0, st));
  eval_kernel_for(P->D)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_ONLY, P->x_tmp.p);
  CK(cudaEventRecord(e1, st));
  CK(cudaGetLastError());
  auto pull = [&](void* dst, const void* src, size_t n) {
    if (!dst || n == 0) return cudaSuccess;
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, st);
  };
  {  // device time and algorithmic bytes of this one full-batch launch (bench.py: roofline of the kernel)
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    P->timing = tb200_timing{};
    P->timing.total_ms = P->timing.convexify_ms = ms;
    P->timing.convexify_launches = 1;
    P->timing.convexify_bytes = 8LL * (dp.N + static_cast<int64_t>(dp.n_coll_cand) * dp.coll_stride +
                                       static_cast<int64_t>(dp.n_cart_rows) * (dp.cart_stride + 1) + dp.n_costs + dp.n_cnts) * dp.B;
  }
  CK(pull(out->cart_err, dp.cart_err, B * dp.n_cart_rows * sizeof(double)));
  CK(pull(out->cart_jac, dp.cart_jac, B * dp.n_cart_rows * dp.cart_stride * sizeof(double)));
  CK(pull(out->coll_rows, dp.coll_rows, B * dp.n_coll_cand * dp.coll_stride * sizeof(double)));
  CK(pull(out->cost_vals, dp.cost_vals, B * dp.n_costs * sizeof(double)));
  CK(pull(out->cnt_viols, dp.cnt_viols, B * dp.n_cnts * sizeof(double)));
  CK(cudaStreamSynchronize(st));
  return lvsOverflowError(P);
}

int tb200_qp_solve_batch(tb200_problem* P, const double* x, const double* trust, const double* merit_coeffs, double* new_x,
                         int32_t* qp_status, double* model_cost_vals, double* model_cnt_viols, int32_t* admm_iters) {
  if (!P || !x || !trust || !merit_coeffs) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  const DevProblem& dp = P->dp;
  const size_t B = dp.B;
  cudaStream_t st = P->stream;
  CK(cudaMemcpyAsync(P->x_tmp.p, x, B * dp.N * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(P->trust_tmp.p, trust, B * sizeof(double), cudaMemcpyHostToDevice, st));
  if (dp.n_cnts > 0) CK(cudaMemcpyAsync(P->merit_coeffs.p, merit_coeffs, B * dp.n_cnts * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(P->ws_meta.p, 0, B * 8 * sizeof(int), st));
  CK(cudaMemsetAsync(P->lvs_overflow.p, 0, B * sizeof(int), st));
  CK(cudaMemsetAsync(P->work_counter.p, 0, sizeof(int), st));
  if (dp.qp_paths) CK(cudaMemsetAsync(dp.qp_paths, 0, B * sizeof(int), st));
  eval_kernel_for(P->D)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_ONLY, P->x_tmp.p);
  SolveCtl ctl{};
  ctl.mode = SOLVE_QP_ONLY;  // one QP step per trajectory (one CTA each), no evaluation / decision
  ctl.quantum = 1;
  ctl.x_override = P->x_tmp.p; ctl.trust_override = P->trust_tmp.p;
  ctl.admm_iters_out = P->tmp_iters.p; ctl.polish_out = P->tmp_polish.p;
  solve_kernel_for(P->D, P->pair_rows)<<<std::min(dp.B, P->n_sm), kQpThreads, P->solve_smem, st>>>(dp, P->ex, ctl);
  CK(cudaGetLastError());
  auto pull = [&](void* dst, const void* src, size_t n) {
    if (!dst || n == 0) return cudaSuccess;
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, st);
  };
  CK(pull(new_x, dp.new_x, B * dp.N * sizeof(double)));
  CK(pull(qp_status, dp.qp_status, B * sizeof(int)));
  CK(pull(model_cost_vals, dp.model_cost_vals, B * dp.n_costs * sizeof(double)));
  CK(pull(model_cnt_viols, dp.model_cnt_viols, B * dp.n_cnts * sizeof(double)));
  CK(pull(admm_iters, P->tmp_iters.p, B * sizeof(int)));
  CK(cudaStreamSynchronize(st));
  return TB200_OK;
}

int tb200_last_qp_polish(tb200_problem* P, int32_t* polish) {
  if (!P || !polish) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(polish, P->tmp_polish.p, static_cast<size_t>(P->dp.B) * sizeof(int), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

/* not part of the public header: enable the per-decision trace (cap entries per trajectory) / fetch it */
int tb200_debug_enable_trace(tb200_problem* P, int cap) {
  if (!P) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  P->trace.release();
  CK(P->trace.alloc(static_cast<size_t>(P->dp.B) * cap * 14));
  P->dp.trace = P->trace.p;
  P->dp.trace_cap = cap;
  return TB200_OK;
}
int tb200_debug_fetch_trace(tb200_problem* P, double* out, int32_t* len) {
  if (!P || !out || !len) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(out, P->trace.p, P->trace.n * sizeof(double), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(len, P->trace_len.p, static_cast<size_t>(P->dp.B) * sizeof(int), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

int tb200_debug_prof(unsigned long long* out, int reset) { return qp_debug_prof(out, reset); }
int tb200_debug_eval_prof(unsigned long long* out, int reset) { return eval_debug_prof(out, reset); }

/* not part of the public header: schedule of the last solve: out[0] = first claim (ns), out[1 + b] = finish time of
   trajectory b (ns), out[1 + B + b] = ns it was being worked on */
int tb200_debug_schedule(tb200_problem* P, unsigned long long* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  const size_t B = P->dp.B;
  CK(cudaMemcpy(out, P->sched_timers.p + 4, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(out + 1, P->sched_timers.p + 8, 2 * B * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

/* not part of the public header: the time limit of the last solve: *start_ns = %globaltimer at its start (the clock
   the limit is measured on, comparable with tb200_debug_schedule's times), ended[b] = what ended trajectory b:
   1 the limit, 2 its group (group_stop), 0 its own SQP */
int tb200_debug_time_limit(tb200_problem* P, unsigned long long* start_ns, int32_t* ended) {
  if (!P || !start_ns || !ended) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(start_ns, P->clock_start.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ended, P->ended_by.p, static_cast<size_t>(P->dp.B) * sizeof(int), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

/* not part of the public header: the group flags of the last solve, done[g] = 1 when a seed of group g ended
   OPT_CONVERGED by its own SQP while group_stop was on; [batch / group_size] */
int tb200_debug_group_done(tb200_problem* P, int32_t* done) {
  if (!P || !done) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  if (P->solved_group_size == 0) return fail(TB200_ERR_INVALID, "no solve yet");
  CK(cudaMemcpy(done, P->group_done.p, static_cast<size_t>(P->dp.B / P->solved_group_size) * sizeof(int), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

/* not part of the public header: record which code paths the QP solver takes (QpPath bits of qp_cta_kernel.cuh), on = 1,
   or stop recording (on = 0, the default); then out[b] = the bits of every QP of trajectory b since the start of the last
   tb200_solve_batch* / tb200_qp_solve_batch */
int tb200_debug_enable_qp_paths(tb200_problem* P, int on) {
  if (!P) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  if (on && !P->qp_paths.p) CK(P->qp_paths.alloc(static_cast<size_t>(P->dp.B)));
  P->dp.qp_paths = on ? P->qp_paths.p : nullptr;
  return TB200_OK;
}
/* not part of the public header, no device needed: the layout the QP step takes for a problem of n_steps waypoints of
   n_dof joints whose QP rows span two waypoints (pair_rows) or one, with at most max_rows rows; a QP whose rows fit
   shared memory, the default passes.  out[0] blocks M, [1] factor in global memory, [2] band in global memory,
   [3] row_cap, [4] the ADMM block (QpPath bit), [5] 1: the fused check, [6] 1: polish_passes, [7] 1: partition
   inverse planned (qp_smem_layout's pinv) */
int tb200_debug_qp_layout(int n_steps, int n_dof, int pair_rows, int max_rows, int32_t* out) {
  if (!out || n_steps < 1 || n_dof < 1 || n_dof > TB200_MAX_DOF || max_rows < 1) return fail(TB200_ERR_INVALID, "bad argument");
  const int N = n_steps * n_dof, nb = 2 * n_dof;
  const int CN = pair_rows ? std::max(2 * n_dof, 3) : std::max(n_dof, 3);
  const bool fg = n_dof > 8;  // = FG of qp_step
  const QpSmem s = qp_smem_layout(N, nb, qp_row_stride(CN), CN, max_rows, fg);
  const int M = qp_block_count(N, nb);
  const QpPlan pl = qp_plan(n_dof <= 7, s.pinv, 1, M, nb, true);
  out[0] = M;
  out[1] = (fg || !s.factor_smem) ? 1 : 0;
  out[2] = s.pband_smem ? 0 : 1;
  out[3] = s.row_cap;
  out[4] = qp_plan_block(pl, 1);
  out[5] = pl.fuse ? 1 : 0;
  out[6] = pl.fast_polish ? 1 : 0;
  out[7] = s.pinv;
  return TB200_OK;
}
int tb200_debug_qp_paths(tb200_problem* P, int32_t* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  if (!P->dp.qp_paths) return fail(TB200_ERR_INVALID, "QP path recording is off (tb200_debug_enable_qp_paths)");
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(out, P->qp_paths.p, static_cast<size_t>(P->dp.B) * sizeof(int), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

/* not part of the public header: solver diagnostics of the last QP of every trajectory, [B][16] */
int tb200_debug_last_qp(tb200_problem* P, double* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(out, P->dbg.p, static_cast<size_t>(P->dp.B) * 16 * sizeof(double), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

int tb200_check_trajectories(tb200_problem* P, const double* x, const tb200_check_config* cfg, tb200_check_results* out) {
  if (!P || !cfg || !out) return fail(TB200_ERR_INVALID, "null argument");
  const int type = cfg->type;
  if (type != TB200_COLL_DISCRETE && type != TB200_COLL_LVS_DISCRETE && type != TB200_COLL_CONTINUOUS &&
      type != TB200_COLL_LVS_CONTINUOUS)
    return fail(TB200_ERR_INVALID, "unknown collision check type " + std::to_string(type) +
                                       " (1 DISCRETE, 2 LVS_DISCRETE, 3 CONTINUOUS, 4 LVS_CONTINUOUS)");
  if ((type == TB200_COLL_LVS_DISCRETE || type == TB200_COLL_LVS_CONTINUOUS) && !(cfg->longest_valid_segment_length > 0.0))
    return fail(TB200_ERR_INVALID, "longest_valid_segment_length must be > 0 for the LVS check types");
  if (!std::isfinite(cfg->margin)) return fail(TB200_ERR_INVALID, "the check margin must be finite");
  if (!x && P->solved_group_size == 0) return fail(TB200_ERR_INVALID, "x is NULL and there is no solve whose result could be checked");
  CK(cudaSetDevice(P->device));
  const DevProblem& dp = P->dp;
  const size_t B = dp.B, T = dp.T;
  if (!P->chk_min.p) {
    CK(P->chk_slot_min.alloc(B * T)); CK(P->chk_slot_contacts.alloc(B * T)); CK(P->chk_slot_argmin.alloc(B * T * 3));
    CK(P->chk_in_collision.alloc(B)); CK(P->chk_first.alloc(B)); CK(P->chk_min.alloc(B));
  }
  cudaStream_t st = P->stream;
  if (x) CK(cudaMemcpyAsync(P->x_tmp.p, x, B * dp.N * sizeof(double), cudaMemcpyHostToDevice, st));
  CheckArgs a{};
  a.segs = dp.segs; a.spheres = dp.spheres; a.obstacles = dp.obstacles;
  a.x = x ? P->x_tmp.p : dp.x;  // NULL: the iterates the last solve left on the device
  a.B = dp.B; a.T = dp.T; a.D = dp.D; a.S = dp.S; a.L = dp.L; a.O = dp.O; a.obstacles_per_traj = dp.obstacles_per_traj;
  a.type = type;
  a.n_slots = (type == TB200_COLL_DISCRETE) ? dp.T : dp.T - 1;
  a.lvs = cfg->longest_valid_segment_length;
  a.margin = cfg->margin;
  a.slot_min = P->chk_slot_min.p; a.slot_contacts = P->chk_slot_contacts.p; a.slot_argmin = P->chk_slot_argmin.p;
  a.in_collision = P->chk_in_collision.p; a.first_slot = P->chk_first.p; a.min_distance = P->chk_min.p;
  CK(launch_check_trajectories(a, P->n_sm, st));
  const size_t S = a.n_slots;
  auto pull = [&](void* dst, const void* src, size_t n) {
    return (dst && n) ? cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, st) : cudaSuccess;
  };
  CK(pull(out->step_min_distance, a.slot_min, B * S * sizeof(double)));
  CK(pull(out->step_contacts, a.slot_contacts, B * S * sizeof(int)));
  CK(pull(out->step_argmin, a.slot_argmin, B * S * 3 * sizeof(int)));
  CK(pull(out->in_collision, a.in_collision, B * sizeof(int)));
  CK(pull(out->first_slot, a.first_slot, B * sizeof(int)));
  CK(pull(out->min_distance, a.min_distance, B * sizeof(double)));
  CK(cudaStreamSynchronize(st));
  return TB200_OK;
}

int tb200_problem_set_sqp_log(tb200_problem* P, int32_t capacity, int32_t with_x) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  if (capacity < 0) return fail(TB200_ERR_INVALID, "sqp log capacity must be >= 0 (0: off)");
  if (with_x != 0 && with_x != 1) return fail(TB200_ERR_INVALID, "with_x must be 0 or 1");
  // the whole buffer, [batch][capacity][stride] doubles, must be addressable (and its int stride representable)
  const size_t stride = logStride(P, with_x), limit = std::numeric_limits<size_t>::max() / sizeof(double);
  if (stride > static_cast<size_t>(INT_MAX) ||
      (capacity > 0 && static_cast<size_t>(capacity) > limit / stride / static_cast<size_t>(P->B)))
    return fail(TB200_ERR_INVALID, "sqp log of " + std::to_string(capacity) + " records per trajectory is too large");
  P->log_cap_next = capacity;
  P->log_with_x_next = capacity > 0 ? with_x : 0;
  return TB200_OK;
}

int tb200_fetch_sqp_log(tb200_problem* P, tb200_sqp_log* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  if (!P->log_solved) return fail(TB200_ERR_INVALID, "the last solve ran without the SQP log (tb200_problem_set_sqp_log)");
  const DevProblem& dp = P->dp;
  const EvalExtra& ex = P->ex;
  if (out->new_x && !ex.log_with_x) return fail(TB200_ERR_INVALID, "new_x requested, but the log was recorded without x");
  CK(cudaSetDevice(P->device));
  const size_t B = dp.B, R = ex.log_cap, S = ex.log_stride, nc = dp.n_costs, nk = dp.n_cnts, N = dp.N;
  std::vector<double> raw(B * R * S);
  std::vector<int32_t> len(B), dropped(B);
  CK(cudaMemcpyAsync(raw.data(), P->log.p, raw.size() * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
  CK(cudaMemcpyAsync(len.data(), P->log_len.p, B * sizeof(int), cudaMemcpyDeviceToHost, P->stream));
  CK(cudaMemcpyAsync(dropped.data(), P->log_dropped.p, B * sizeof(int), cudaMemcpyDeviceToHost, P->stream));
  CK(cudaStreamSynchronize(P->stream));
  const double qnan = std::numeric_limits<double>::quiet_NaN();
  for (size_t b = 0; b < B; ++b) {
    if (out->n_records) out->n_records[b] = len[b];
    if (out->n_dropped) out->n_dropped[b] = dropped[b];
    const double* old = nullptr;  // exact values of the last accepted point: the record of kind 0 or the last accept
    for (size_t r = 0; r < R; ++r) {
      const size_t i = b * R + r;
      const bool have = static_cast<int>(r) < len[b];
      const double* h = raw.data() + i * S;
      const double* mu = h + kLogHeader;
      const double *mc = mu + nk, *mk = mc + nc, *vc = mk + nk, *vk = vc + nc, *x = vk + nk;
      auto put_i = [&](int32_t* dst, int f) { if (dst) dst[i] = have ? static_cast<int32_t>(h[f]) : 0; };
      auto put_d = [&](double* dst, int f) { if (dst) dst[i] = have ? h[f] : qnan; };
      auto put_v = [&](double* dst, const double* src, size_t n) {
        if (dst) for (size_t k = 0; k < n; ++k) dst[i * n + k] = (have && src) ? src[k] : qnan;
      };
      put_i(out->kind, LOG_KIND); put_i(out->merit_round, LOG_ROUND); put_i(out->iter, LOG_ITER);
      put_d(out->trust_box_size, LOG_TRUST);
      put_d(out->old_merit, LOG_OLD_MERIT); put_d(out->model_merit, LOG_MODEL_MERIT); put_d(out->new_merit, LOG_NEW_MERIT);
      put_i(out->action, LOG_ACTION); put_i(out->ended, LOG_ENDED);
      const bool qp = have && h[LOG_KIND] == 1;
      if (out->qp_status) out->qp_status[i] = qp ? static_cast<int32_t>(h[LOG_QP_STATUS]) : -1;
      if (out->admm_iters) out->admm_iters[i] = qp ? static_cast<int32_t>(h[LOG_ADMM_ITERS]) : 0;
      if (out->polish) out->polish[i] = qp ? static_cast<int32_t>(h[LOG_POLISH]) : 0;
      if (out->qp_diag)
        for (int k = 0; k < 4; ++k) out->qp_diag[i * 4 + k] = qp ? h[(k < 3 ? LOG_PRI_RES + k : LOG_WARM)] : qnan;
      put_v(out->merit_coeffs, mu, nk);
      put_v(out->model_cost_vals, mc, nc); put_v(out->model_cnt_viols, mk, nk);
      put_v(out->new_cost_vals, vc, nc); put_v(out->new_cnt_viols, vk, nk);
      put_v(out->old_cost_vals, qp ? old : nullptr, nc);
      put_v(out->old_cnt_viols, qp ? (old ? old + nc : nullptr) : nullptr, nk);
      if (out->new_x) put_v(out->new_x, x, N);
      if (have && (h[LOG_KIND] == 0 || h[LOG_ACTION] == 1)) old = vc;  // (vc, vk are adjacent)
    }
  }
  return TB200_OK;
}

int tb200_problem_objects(const tb200_problem* P, int32_t* term, int32_t* step) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  for (size_t i = 0; i < P->obj_src.size(); ++i) {
    if (term) term[i] = P->obj_src[i].first;
    if (step) step[i] = P->obj_src[i].second;
  }
  return TB200_OK;
}

int tb200_last_timing(const tb200_problem* p, tb200_timing* out) {
  if (!p || !out) return fail(TB200_ERR_INVALID, "null argument");
  *out = p->timing;
  return TB200_OK;
}

}  // extern "C"
