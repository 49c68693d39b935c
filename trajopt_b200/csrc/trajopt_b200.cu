// Host side of the C ABI (include/trajopt_b200.h): creates a problem from its flattened description (flatten.h), owns
// the device buffers, and drives the batched trust-region SQP (trajopt_sco/src/optimizers.cpp:699-991): one launch of
// eval_convexify_decide_kernel (first evaluation + convexification of every trajectory) and one persistent launch of
// solve_kernel, which runs every trajectory's QP subproblems, merit evaluations, re-convexifications and
// accept/shrink/penalty decisions.
// CUDA only: every entry point fails with TB200_ERR_CUDA / TB200_ERR_NO_DEVICE when no device is usable.
#include <cuda_runtime.h>
#include <math_constants.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "../../include/trajopt_b200.h"
#include "check_kernel.cuh"
#include "dev_buf.h"
#include "eval_kernel.cuh"
#include "flatten.h"
#include "solve_kernel.cuh"
#include "kernels.h"

using namespace tb200;

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

// G = 0 and G = 1 are both "no groups": every trajectory is its own group and nothing is stopped
void setGroups(DevProblem& dp, int group_size, int group_stop) {
  dp.group_size = std::max(group_size, 1);
  dp.group_stop = dp.group_size > 1 ? group_stop : 0;
}
}  // namespace

struct tb200_problem {
  int device = 0;
  DevProblem dp{};
  EvalExtra ex{};
  int B = 0, T = 0, D = 0, N = 0;
  size_t eval_smem = 0, qp_smem = 0, solve_smem = 0;
  int n_sm = 132;  // H100 SXM; replaced by the device's own count at problem creation
  int quantum = 3;  // SQP steps a CTA runs of a trajectory before it looks for a more urgent one (TB200_QUANTUM overrides)
  cudaStream_t stream = nullptr;
  tb200_timing timing{};
  std::vector<std::pair<int, int>> obj_src;  // per object (costs, then constraints): the term that hatched it, its step
  // SQP iteration log: the setting of the next solve, and the buffers of the last one (log_solved: it ran with the log)
  int log_cap_next = 0, log_with_x_next = 0;
  bool log_solved = false;
  DevBuf<double> log;
  DevBuf<int> log_len, log_dropped;
  bool pair_rows = false;  // QP rows span two waypoints (CartVel, continuous collision): 2*D coefficients per row
  bool sing = false;       // AvoidSingularity objects: the kernel instances with the term (SING = 1)
  // optimizer parameters: the uniform ones (tb200_problem_set_sqp_params), and the [B] rows the kernels read (EvalExtra::sqp),
  // the uniform ones in every row unless a per-trajectory table was given
  tb200_sqp_params sqp_uniform{};
  DevBuf<SqpParams> sqp_rows;
  // device storage
  DevBuf<DevSegment> segs;
  DevBuf<DevSphere> spheres;
  DevBuf<double> lower, upper, Pband, qlin, init_traj, cart_targets, obstacles;
  DevBuf<DevObj> d_cost_objs, d_cnt_objs, d_cart_objs, d_coll_objs, d_vel_objs, d_sing_objs;
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
  std::vector<cudaEvent_t> events;
  ~tb200_problem() {  // (the buffers free themselves)
    for (auto e : events) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace {
// Queues a copy of n bytes from the device to the caller on the problem's stream; a NULL destination (or n = 0) is
// skipped, and a copy that is made adds n to *bytes when bytes is given.
cudaError_t pull(tb200_problem* P, void* dst, const void* src, size_t n, int64_t* bytes = nullptr) {
  if (!dst || n == 0) return cudaSuccess;
  if (bytes) *bytes += static_cast<int64_t>(n);
  return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, P->stream);
}

// Copies n elements of a device buffer to the caller, synchronously (the tb200_debug_* getters).
template <class T>
int copyOut(tb200_problem* P, T* dst, const T* src, size_t n) {
  CK(cudaSetDevice(P->device));
  CK(cudaMemcpy(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost));
  return TB200_OK;
}

// Algorithmic HBM bytes of convexifying one trajectory (SURVEY.md §8d): read x, write cart rows, dense collision rows
// and the exact values.
int64_t convexifyBytes(const DevProblem& dp) {
  return 8LL * (dp.N + static_cast<int64_t>(dp.n_coll_cand) * dp.coll_stride +
                static_cast<int64_t>(dp.n_cart_rows) * (dp.cart_stride + 1) + dp.n_costs + dp.n_cnts);
}

// The sizes and tables of DevProblem / EvalExtra and the kernels' shared memory, from the flattened description; refuses
// a problem no kernel instance can run.
int planLayout(const tb200_problem_desc& d, const FlatProblem& F, tb200_problem& P) {
  const int T = d.n_steps, D = d.robot.n_dof, B = d.batch, N = T * D;
  P.B = B; P.T = T; P.D = D; P.N = N;
  DevProblem& dp = P.dp;
  dp.B = B; dp.T = T; dp.D = D; dp.N = N; dp.HB = 2 * D;
  dp.S = static_cast<int>(F.segs.size()); dp.L = d.robot.n_spheres; dp.O = d.n_obstacles;
  dp.obstacles_per_traj = d.obstacles_per_traj;
  dp.n_cart_targets = d.n_cart_targets;
  dp.n_band = F.n_band;
  std::copy(std::begin(F.band_offs), std::end(F.band_offs), dp.band_offs);
  dp.n_costs = static_cast<int>(F.cost_objs.size());
  dp.n_cnts = static_cast<int>(F.cnt_objs.size());
  dp.n_cart_rows = F.n_cart_rows;
  const int CN = (F.has_vel || F.has_cast) ? std::max(2 * D, 3) : std::max(D, 3);  // coefficients per (padded) QP row
  dp.cart_stride = F.has_vel ? 2 * D : D;
  dp.n_coll_cand = F.n_coll_cand;
  dp.coll_stride = F.has_cast ? 2 * D + 3 : D + 3;
  dp.n_fixed = static_cast<int>(F.fixed_vars.size());
  dp.max_rows = F.max_rows;
  dp.row_stride = qp_row_stride(CN);
  dp.coll_words = std::max(1, ((F.has_cast ? F.cast_cap : dp.L * dp.O) + 63) / 64);
  dp.n_coll_objs = static_cast<int>(F.coll_objs.size());
  dp.qp = QpSettings{d.qp.rho, d.qp.sigma, d.qp.alpha, d.qp.eps_abs, d.qp.eps_rel, d.qp.eps_prim_inf, d.qp.eps_dual_inf,
                     d.qp.delta, d.qp.adaptive_rho_tolerance, d.qp.max_iter, d.qp.scaling, d.qp.check_termination,
                     d.qp.adaptive_rho, d.qp.adaptive_rho_interval, d.qp.polishing, d.qp.polish_refine_iter,
                     d.qp.warm_starting, d.qp.early_polish_every, d.qp.early_polish_from};
  P.sqp_uniform = d.sqp;
  setGroups(dp, d.group_size, d.group_stop);
  EvalExtra& ex = P.ex;
  ex.n_cart_objs = static_cast<int>(F.cart_objs.size());
  ex.n_coll_objs = dp.n_coll_objs;
  ex.n_vel_objs = static_cast<int>(F.vel_objs.size());
  ex.n_sing_objs = static_cast<int>(F.sing_objs.size());
  P.sing = ex.n_sing_objs > 0;
  ex.cast = F.has_cast ? 1 : 0;
  ex.cast_cap = F.cast_cap;
  ex.n_joint_objs = F.n_joint_objs;
  std::copy(std::begin(F.joint_obj_idx), std::end(F.joint_obj_idx), ex.joint_obj_idx);
  std::copy(std::begin(F.joint_seg), std::end(F.joint_seg), ex.joint_seg);
  std::copy(std::begin(F.qtype), std::end(F.qtype), ex.qtype);
  std::copy(std::begin(F.sphere_jmask), std::end(F.sphere_jmask), ex.sphere_jmask);

  const EvalSmem es = eval_smem_layout(T, D, dp.L, dp.n_coll_objs, dp.n_coll_objs * dp.coll_words, dp.S, ex.n_joint_objs,
                                       ex.n_vel_objs, ex.cast, ex.cast_cap, dp.n_costs + dp.n_cnts, ex.n_sing_objs);
  P.pair_rows = F.has_vel || F.has_cast;  // (at one joint such rows still fit the 3 padded coefficients of a row)
  P.eval_smem = static_cast<size_t>(es.total) * sizeof(double);
  const bool factor_global = D > 8;  // = FG of qp_step: blocks of 2*D > 16 never fit
  const QpSmem qs = qp_smem_layout(N, 2 * D, dp.row_stride, CN, dp.max_rows, factor_global);
  const int Np = qp_block_count(N, 2 * D) * 2 * D;
  dp.list_stride = static_cast<size_t>(Np + 1) + static_cast<size_t>(dp.max_rows) * CN + dp.n_costs + dp.n_cnts + 2;
  dp.soa_stride = (dp.max_rows > qs.row_cap) ? qp_soa_doubles(dp.max_rows, CN) : 0;
  P.qp_smem = static_cast<size_t>(qs.total) * sizeof(double);
  if (P.eval_smem > 226 * 1024 || P.qp_smem > 226 * 1024)
    return fail(TB200_ERR_UNSUPPORTED, "problem does not fit the 227 KB shared memory of one CTA");
  if (CN > 32) return fail(TB200_ERR_UNSUPPORTED, "more than 32 coefficients per QP row");
  if (!solve_kernel_for(D, P.pair_rows, P.sing) || !eval_kernel_for(D, P.sing))
    return fail(TB200_ERR_UNSUPPORTED, P.pair_rows ? "no kernel instance with two-waypoint rows (CartVel, continuous collision) for this number of joints"
                                                   : "no kernel instance for this number of joints");
  return TB200_OK;
}

// The device, its limits and the kernels' attributes, the solver's stream and the grid of a stand-alone evaluation.
int setupDevice(tb200_problem& P, int device) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(TB200_ERR_NO_DEVICE, "no CUDA device: trajopt_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(TB200_ERR_INVALID, "bad device ordinal");
  P.device = device;
  CK(cudaSetDevice(device));
  {  // the QP step calls its hot functions through pointers (standard calling convention): make sure the per-thread stack
     // covers the deepest chain (ptxas reports < 3 KB for the chains it can follow)
    size_t cur = 0;
    CK(cudaDeviceGetLimit(&cur, cudaLimitStackSize));
    if (cur < 6144) CK(cudaDeviceSetLimit(cudaLimitStackSize, 6144));
  }
  CK(cudaFuncSetAttribute(eval_kernel_for(P.D, P.sing), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P.eval_smem)));
  P.solve_smem = std::max(P.qp_smem, P.eval_smem);  // the QP step and the evaluation step share one buffer
  CK(cudaFuncSetAttribute(solve_kernel_for(P.D, P.pair_rows, P.sing), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P.solve_smem)));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  P.n_sm = std::max(1, sms);
  int per_sm = 1;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, eval_kernel_for(P.D, P.sing), kEvalThreads, P.eval_smem));
  P.eval_grid = std::max(1, std::min(P.B, std::max(1, per_sm) * P.n_sm));
  if (const char* e = std::getenv("TB200_QUANTUM")) P.quantum = std::max(1, std::atoi(e));
  // TB200_GENERIC_QP_PASSES=1: termination checks and polish refinement by the generic passes of the QP solver instead
  // of the check fused into the ADMM block and polish_passes (same decisions; the switch exists to compare the two)
  const char* generic = std::getenv("TB200_GENERIC_QP_PASSES");
  P.dp.qp_fast_passes = (generic && std::atoi(generic) != 0) ? 0 : 1;
  CK(cudaStreamCreateWithFlags(&P.stream, cudaStreamNonBlocking));
  return TB200_OK;
}

// Allocates every device buffer of the problem, uploads the flattened tables and points DevProblem / EvalExtra at them.
int allocate(const tb200_problem_desc& d, FlatProblem& F, tb200_problem& P) {
  DevProblem& dp = P.dp;
  EvalExtra& ex = P.ex;
  cudaError_t e = cudaSuccess;  // the first failure; the buffers after it are not allocated
  auto zeros = [&](auto& buf, size_t count) {
    if (e == cudaSuccess) e = buf.alloc(count);
    return buf.p;
  };
  auto upload = [&](auto& buf, const auto& v) {
    zeros(buf, v.size());
    if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(buf.p, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
    return buf.p;
  };
  const int D = P.D;
  const size_t B = P.B, N = P.N, Np = static_cast<size_t>(qp_block_count(P.N, 2 * D)) * 2 * D;
  const size_t n_costs = std::max(1, dp.n_costs), n_cnts = std::max(1, dp.n_cnts), max_rows = dp.max_rows;
  dp.segs = upload(P.segs, F.segs);
  dp.spheres = upload(P.spheres, F.spheres);
  dp.lower = upload(P.lower, std::vector<double>(d.robot.lower, d.robot.lower + D));
  dp.upper = upload(P.upper, std::vector<double>(d.robot.upper, d.robot.upper + D));
  dp.Pband = upload(P.Pband, F.Pband);
  dp.qlin = upload(P.qlin, F.qlin);
  dp.cost_objs = upload(P.d_cost_objs, F.cost_objs);
  dp.cnt_objs = upload(P.d_cnt_objs, F.cnt_objs);
  ex.cart_objs = upload(P.d_cart_objs, F.cart_objs);
  ex.coll_objs = upload(P.d_coll_objs, F.coll_objs);
  ex.vel_objs = upload(P.d_vel_objs, F.vel_objs);
  ex.sing_objs = upload(P.d_sing_objs, F.sing_objs);
  dp.joint_terms = upload(P.joint_terms, F.joint_terms);
  dp.cart_terms = upload(P.cart_terms, F.cart_terms);
  dp.fixed_vars = upload(P.fixed_vars, F.fixed_vars);
  ex.link_chain = upload(P.link_chain, F.link_chain);
  dp.init_traj = zeros(P.init_traj, B * N);
  dp.cart_targets = zeros(P.cart_targets, B * std::max(1, d.n_cart_targets) * 7);
  dp.obstacles = zeros(P.obstacles, (d.obstacles_per_traj ? B : 1) * std::max(1, dp.O) * 4);
  dp.x = zeros(P.x, B * N); dp.new_x = zeros(P.new_x, B * N); dp.trust = zeros(P.trust, B);
  dp.merit_coeffs = zeros(P.merit_coeffs, B * n_cnts);
  dp.cost_vals = zeros(P.cost_vals, B * n_costs); dp.cnt_viols = zeros(P.cnt_viols, B * n_cnts);
  dp.new_cost_vals = zeros(P.new_cost_vals, B * n_costs); dp.new_cnt_viols = zeros(P.new_cnt_viols, B * n_cnts);
  dp.model_cost_vals = zeros(P.model_cost_vals, B * n_costs); dp.model_cnt_viols = zeros(P.model_cnt_viols, B * n_cnts);
  dp.cart_err = zeros(P.cart_err, 2 * B * std::max(1, dp.n_cart_rows));
  dp.cart_jac = zeros(P.cart_jac, 2 * B * std::max(1, dp.n_cart_rows) * dp.cart_stride);
  dp.coll_rows = zeros(P.coll_rows, 2 * B * std::max(1, dp.n_coll_cand) * dp.coll_stride);
  dp.coll_mask = zeros(P.coll_mask, 2 * B * std::max(1, dp.n_coll_objs * dp.coll_words));
  dp.rows = zeros(P.rows, B * max_rows * dp.row_stride); dp.row_ints = zeros(P.row_ints, B * max_rows * RI_NINTS);
  dp.lists = zeros(P.lists, B * dp.list_stride);
  dp.ws_x = zeros(P.ws_x, B * N); dp.ws_yb = zeros(P.ws_yb, B * N); dp.scratch = zeros(P.scratch, B * 5 * Np);
  dp.qp_done = zeros(P.qp_done, B); dp.ws_rho = zeros(P.ws_rho, B); dp.ws_meta = zeros(P.ws_meta, B * 8);
  dp.lvs_overflow = zeros(P.lvs_overflow, B);
  ex.work_counter = zeros(P.work_counter, 1);
  ex.sqp = zeros(P.sqp_rows, B);
  // contact lists of the continuous collision evaluator: one per resident warp of the largest launch (4 doubles a contact)
  ex.cast_scratch = zeros(P.cast_scratch, ex.cast ? static_cast<size_t>(std::max(P.eval_grid, std::min(P.B, P.n_sm))) *
                                                        (kEvalThreads / 32) * 4 * ex.cast_cap : 0);
  // per-CTA regions (the persistent kernel and the kernel-level QP entry point both launch at most one CTA per SM):
  // the factor of wide blocks or the rows of the partition inverses, and the column-major copy of rows that do not fit
  // shared memory
  dp.factor_g = zeros(P.factor_g, static_cast<size_t>(P.n_sm) * qp_cta_global_doubles(P.N, 2 * D));
  dp.soa = zeros(P.soa, static_cast<size_t>(P.n_sm) * dp.soa_stride);
  dp.status = zeros(P.status, B); dp.sqp_iter = zeros(P.sqp_iter, B); dp.merit_round = zeros(P.merit_round, B);
  dp.qp_failures = zeros(P.qp_failures, B); dp.qp_status = zeros(P.qp_status, B); dp.cur_buf = zeros(P.cur_buf, B);
  dp.n_qp_solves = zeros(P.n_qp_solves, B); dp.n_func_evals = zeros(P.n_func_evals, B);
  dp.n_admm_iters = zeros(P.n_admm_iters, B);
  dp.active_count = zeros(P.active_count, 2);
  dp.dbg = zeros(P.dbg, B * 16);
  dp.sched_state = zeros(P.sched_state, B); dp.sched_timers = zeros(P.sched_timers, 8 + 2 * B);
  dp.clock_start = zeros(P.clock_start, 1); dp.sqp_top = zeros(P.sqp_top, B); dp.ended_by = zeros(P.ended_by, B);
  dp.group_done = zeros(P.group_done, B);
  dp.trace_len = zeros(P.trace_len, B);
  zeros(P.g_best, B); zeros(P.g_status, B); zeros(P.g_n_converged, B); zeros(P.g_total_cost, B); zeros(P.g_x, B * N);
  zeros(P.x_tmp, B * N); zeros(P.trust_tmp, B); zeros(P.tmp_iters, B); zeros(P.tmp_polish, B);
  if (e != cudaSuccess) return fail(TB200_ERR_CUDA, std::string("device buffers of the problem: ") + cudaGetErrorString(e));
  // the zero fills (cudaMemset, asynchronous on the legacy stream) end before the uploads on the solver's non-blocking
  // stream, which does not wait for them
  CK(cudaDeviceSynchronize());
  P.obj_src = std::move(F.obj_src);
  return TB200_OK;
}

// Uploads the optimizer parameters of the next solves, row b for trajectory b, and whether any row has a time limit.
int uploadSqpRows(tb200_problem& P, const std::vector<SqpParams>& rows) {
  CK(cudaSetDevice(P.device));
  CK(cudaMemcpyAsync(P.sqp_rows.p, rows.data(), rows.size() * sizeof(SqpParams), cudaMemcpyHostToDevice, P.stream));
  CK(cudaStreamSynchronize(P.stream));
  P.ex.sqp_timed = std::any_of(rows.begin(), rows.end(), [](const SqpParams& r) { return r.max_time < kNoTimeLimit; });
  return TB200_OK;
}

}  // namespace

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
  // the description is checked and flattened first - pure host work, so that a bad description gets the same error
  // with or without a device - and only then the device is touched
  FlatProblem F;
  std::string msg;
  if (int rc = flatten(*d, F, msg)) return fail(rc, msg);
  auto P = std::make_unique<tb200_problem>();
  if (int rc = planLayout(*d, F, *P)) return rc;
  if (int rc = setupDevice(*P, device)) return rc;
  if (int rc = allocate(*d, F, *P)) return rc;
  if (int rc = uploadSqpRows(*P, F.sqp_rows)) return rc;
  if (int rc = tb200_problem_set_inputs(P.get(), d->init_traj, d->cart_targets, d->obstacles)) return rc;
  *out = P.release();
  return TB200_OK;
}

void tb200_problem_destroy(tb200_problem* p) { delete p; }

int tb200_problem_layout(const tb200_problem* p, tb200_layout* out) {
  if (!p || !out) return fail(TB200_ERR_INVALID, "null argument");
  const DevProblem& dp = p->dp;
  *out = tb200_layout{dp.n_costs, dp.n_cnts, dp.n_cart_rows, dp.cart_stride, dp.n_coll_cand, dp.coll_stride, dp.N, 0};
  return TB200_OK;
}

int tb200_problem_set_sqp_params(tb200_problem* P, const tb200_sqp_params* s) {
  if (!P || !s) return fail(TB200_ERR_INVALID, "null argument");
  P->sqp_uniform = *s;
  return uploadSqpRows(*P, flat::sqp_rows(P->B, *s, nullptr));
}

int tb200_problem_set_sqp_params_per_traj(tb200_problem* P, const tb200_sqp_params* rows) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  return uploadSqpRows(*P, flat::sqp_rows(P->B, P->sqp_uniform, rows));
}

int tb200_problem_set_groups(tb200_problem* P, int32_t group_size, int32_t group_stop) {
  if (!P) return fail(TB200_ERR_INVALID, "null problem");
  std::string msg;
  if (int rc = flat::check_groups(P->B, group_size, group_stop, msg)) return fail(rc, msg);
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
__global__ void reset_state_kernel(DevProblem p, const SqpParams* sqp, int* log_len, int* log_dropped) {
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
  p.trust[b] = sqp[b].trust_box_size;
  for (int c = 0; c < p.n_cnts; ++c) p.merit_coeffs[static_cast<size_t>(b) * p.n_cnts + c] = sqp[b].initial_merit_error_coeff;
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
  reset_state_kernel<<<(dp.B + 127) / 128, 128, 0, st>>>(dp, P->ex.sqp, P->ex.log_len, P->ex.log_dropped);
  if (dp.qp_paths) CK(cudaMemsetAsync(dp.qp_paths, 0, dp.B * sizeof(int), st));
  // the initial evaluation + convexification of every trajectory: one CTA per trajectory (optimizers.cpp:761-783)
  CK(cudaEventRecord(e_init0, st));
  CK(cudaMemsetAsync(P->work_counter.p, 0, sizeof(int), st));
  eval_kernel_for(P->D, P->sing)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_INIT, nullptr);
  CK(cudaEventRecord(e_init1, st));
  // everything else: one persistent CTA per SM (solve_kernel.cuh); no host round trips until every trajectory is done
  SolveCtl ctl{};
  ctl.mode = SOLVE_FULL;
  ctl.quantum = P->quantum;
  ctl.sched_state = dp.sched_state;
  ctl.timers = dp.sched_timers;
  solve_kernel_for(P->D, P->pair_rows, P->sing)<<<std::min(dp.B, P->n_sm), kQpThreads, P->solve_smem, st>>>(dp, P->ex, ctl);
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
  int counters[2] = {0, 0};  // trajectories still active, trajectories convexified (summed over all launches)
  CK(cudaMemcpy(counters, dp.active_count, sizeof(counters), cudaMemcpyDeviceToHost));
  tm.convexify_bytes = convexifyBytes(dp) * counters[1];
  if (counters[0] > 0) return fail(TB200_ERR_CUDA, "the SQP kernel returned with trajectories still active");
  return TB200_OK;
}

namespace {
// trajectories whose step pairs outgrew the LVS candidate layout (they ended OPT_FAILED; never truncated silently)
int lvsOverflowError(tb200_problem* P) {
  if (!P->ex.cast) return TB200_OK;
  std::vector<int> f(P->dp.B);
  CK(cudaMemcpy(f.data(), P->lvs_overflow.p, f.size() * sizeof(int), cudaMemcpyDeviceToHost));
  const long n = std::count_if(f.begin(), f.end(), [](int v) { return v != 0; });
  if (n > 0)
    return fail(TB200_ERR_UNSUPPORTED, std::to_string(n) + " trajectories have a step pair with more than " +
                                           std::to_string(P->ex.cast_cap) + " active continuous-collision contacts (the row block of a pair, "
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
  CK(pull(P, out->x, dp.x, B * dp.N * sizeof(double), &bytes));
  CK(pull(P, out->status, dp.status, B * sizeof(int), &bytes));
  CK(pull(P, out->cost_vals, dp.cost_vals, B * dp.n_costs * sizeof(double), &bytes));
  CK(pull(P, out->cnt_viols, dp.cnt_viols, B * dp.n_cnts * sizeof(double), &bytes));
  CK(pull(P, out->n_qp_solves, dp.n_qp_solves, B * sizeof(int), &bytes));
  CK(pull(P, out->n_func_evals, dp.n_func_evals, B * sizeof(int), &bytes));
  CK(pull(P, out->n_admm_iters, dp.n_admm_iters, B * sizeof(int), &bytes));
  std::vector<double> cv(out->total_cost ? B * std::max(1, dp.n_costs) : 0);
  if (out->total_cost) CK(pull(P, cv.data(), dp.cost_vals, B * dp.n_costs * sizeof(double)));
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
  CK(pull(P, out->best, P->g_best.p, NG * sizeof(int)));
  CK(pull(P, out->status, P->g_status.p, NG * sizeof(int)));
  CK(pull(P, out->total_cost, P->g_total_cost.p, NG * sizeof(double)));
  CK(pull(P, out->x, P->g_x.p, NG * N * sizeof(double)));
  CK(pull(P, out->n_converged, P->g_n_converged.p, NG * sizeof(int)));
  CK(pull(P, out->ended_by, P->ended_by.p, B * sizeof(int)));
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
  eval_kernel_for(P->D, P->sing)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_ONLY, P->x_tmp.p);
  CK(cudaEventRecord(e1, st));
  CK(cudaGetLastError());
  {  // device time and algorithmic bytes of this one full-batch launch (bench.py: roofline of the kernel)
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    P->timing = tb200_timing{};
    P->timing.total_ms = P->timing.convexify_ms = ms;
    P->timing.convexify_launches = 1;
    P->timing.convexify_bytes = convexifyBytes(dp) * dp.B;
  }
  CK(pull(P, out->cart_err, dp.cart_err, B * dp.n_cart_rows * sizeof(double)));
  CK(pull(P, out->cart_jac, dp.cart_jac, B * dp.n_cart_rows * dp.cart_stride * sizeof(double)));
  CK(pull(P, out->coll_rows, dp.coll_rows, B * dp.n_coll_cand * dp.coll_stride * sizeof(double)));
  CK(pull(P, out->cost_vals, dp.cost_vals, B * dp.n_costs * sizeof(double)));
  CK(pull(P, out->cnt_viols, dp.cnt_viols, B * dp.n_cnts * sizeof(double)));
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
  eval_kernel_for(P->D, P->sing)<<<P->eval_grid, kEvalThreads, P->eval_smem, st>>>(dp, P->ex, EVAL_ONLY, P->x_tmp.p);
  SolveCtl ctl{};
  ctl.mode = SOLVE_QP_ONLY;  // one QP step per trajectory (one CTA each), no evaluation / decision
  ctl.quantum = 1;
  ctl.x_override = P->x_tmp.p; ctl.trust_override = P->trust_tmp.p;
  ctl.admm_iters_out = P->tmp_iters.p; ctl.polish_out = P->tmp_polish.p;
  solve_kernel_for(P->D, P->pair_rows, P->sing)<<<std::min(dp.B, P->n_sm), kQpThreads, P->solve_smem, st>>>(dp, P->ex, ctl);
  CK(cudaGetLastError());
  CK(pull(P, new_x, dp.new_x, B * dp.N * sizeof(double)));
  CK(pull(P, qp_status, dp.qp_status, B * sizeof(int)));
  CK(pull(P, model_cost_vals, dp.model_cost_vals, B * dp.n_costs * sizeof(double)));
  CK(pull(P, model_cnt_viols, dp.model_cnt_viols, B * dp.n_cnts * sizeof(double)));
  CK(pull(P, admm_iters, P->tmp_iters.p, B * sizeof(int)));
  CK(cudaStreamSynchronize(st));
  return TB200_OK;
}

int tb200_last_qp_polish(tb200_problem* P, int32_t* polish) {
  if (!P || !polish) return fail(TB200_ERR_INVALID, "null argument");
  return copyOut(P, polish, P->tmp_polish.p, P->dp.B);
}

/* not part of the public header: enable the per-decision trace (cap entries per trajectory) / fetch it */
int tb200_debug_enable_trace(tb200_problem* P, int cap) {
  if (!P) return fail(TB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(P->device));
  CK(P->trace.alloc(static_cast<size_t>(P->dp.B) * cap * 14));
  P->dp.trace = P->trace.p;
  P->dp.trace_cap = cap;
  return TB200_OK;
}
int tb200_debug_fetch_trace(tb200_problem* P, double* out, int32_t* len) {
  if (!P || !out || !len) return fail(TB200_ERR_INVALID, "null argument");
  if (int rc = copyOut(P, out, P->trace.p, P->trace.n)) return rc;
  return copyOut(P, len, P->trace_len.p, P->dp.B);
}

int tb200_debug_prof(unsigned long long* out, int reset) { return qp_debug_prof(out, reset); }
int tb200_debug_eval_prof(unsigned long long* out, int reset) { return eval_debug_prof(out, reset); }

/* not part of the public header: schedule of the last solve: out[0] = first claim (ns), out[1 + b] = finish time of
   trajectory b (ns), out[1 + B + b] = ns it was being worked on */
int tb200_debug_schedule(tb200_problem* P, unsigned long long* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  if (int rc = copyOut(P, out, P->sched_timers.p + 4, 1)) return rc;
  return copyOut(P, out + 1, P->sched_timers.p + 8, 2 * static_cast<size_t>(P->dp.B));
}

/* not part of the public header: the time limit of the last solve: *start_ns = %globaltimer at its start (the clock
   the limit is measured on, comparable with tb200_debug_schedule's times), ended[b] = what ended trajectory b:
   1 the limit, 2 its group (group_stop), 0 its own SQP */
int tb200_debug_time_limit(tb200_problem* P, unsigned long long* start_ns, int32_t* ended) {
  if (!P || !start_ns || !ended) return fail(TB200_ERR_INVALID, "null argument");
  if (int rc = copyOut(P, start_ns, P->clock_start.p, 1)) return rc;
  return copyOut(P, ended, P->ended_by.p, P->dp.B);
}

/* not part of the public header: the group flags of the last solve, done[g] = 1 when a seed of group g ended
   OPT_CONVERGED by its own SQP while group_stop was on; [batch / group_size] */
int tb200_debug_group_done(tb200_problem* P, int32_t* done) {
  if (!P || !done) return fail(TB200_ERR_INVALID, "null argument");
  if (P->solved_group_size == 0) return fail(TB200_ERR_INVALID, "no solve yet");
  return copyOut(P, done, P->group_done.p, P->dp.B / P->solved_group_size);
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
  return copyOut(P, out, P->qp_paths.p, P->dp.B);
}

/* not part of the public header: solver diagnostics of the last QP of every trajectory, [B][16] */
int tb200_debug_last_qp(tb200_problem* P, double* out) {
  if (!P || !out) return fail(TB200_ERR_INVALID, "null argument");
  return copyOut(P, out, P->dbg.p, static_cast<size_t>(P->dp.B) * 16);
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
  CK(pull(P, out->step_min_distance, a.slot_min, B * S * sizeof(double)));
  CK(pull(P, out->step_contacts, a.slot_contacts, B * S * sizeof(int)));
  CK(pull(P, out->step_argmin, a.slot_argmin, B * S * 3 * sizeof(int)));
  CK(pull(P, out->in_collision, a.in_collision, B * sizeof(int)));
  CK(pull(P, out->first_slot, a.first_slot, B * sizeof(int)));
  CK(pull(P, out->min_distance, a.min_distance, B * sizeof(double)));
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
