// ORACLE — TEST INFRASTRUCTURE ONLY.  C entry points (ctypes) over the CPU restatement; consumed by
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg only.
#include <chrono>
#include <cstring>
#include <limits>
#include <string>

#include "trajopt.hpp"
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace oracle;

namespace {
thread_local std::string g_err;
struct Layout {
  int n_costs, n_cnts, n_cart_rows, cart_stride, n_coll_cand, coll_stride;
};
Layout layoutOf(const tb200_problem_desc& d, const TrajProblem& tp) {
  Layout L{};
  L.n_costs = static_cast<int>(tp.cost_names.size());
  L.n_cnts = static_cast<int>(tp.cnt_names.size());
  const int D = d.robot.n_dof;
  bool has_vel = false, has_cast = false;
  for (int k = 0; k < d.n_terms; ++k) {
    const tb200_term& t = d.terms[k];
    if (t.kind == TB200_TERM_CART_POSE) {
      for (int i = 0; i < 3; ++i) L.n_cart_rows += std::fabs(t.pos_coeffs[i]) > 1e-5;
      for (int i = 0; i < 3; ++i) L.n_cart_rows += std::fabs(t.rot_coeffs[i]) > 1e-5;
    } else if (t.kind == TB200_TERM_CART_VEL) {
      L.n_cart_rows += 6 * (t.last_step - t.first_step + 1);
      has_vel = true;
    } else if (t.kind == TB200_TERM_AVOID_SINGULARITY) {
      L.n_cart_rows += t.last_step - t.first_step + 1;
    } else if (t.kind == TB200_TERM_COLLISION) {
      if (t.evaluator_type != TB200_COLL_DISCRETE) {  // one object per step pair, dense over sub-segments
        L.n_coll_cand += (t.last_step - t.first_step) * tb200inl_cast_rows_per_pair(&d);
        has_cast = true;
        continue;
      }
      int steps = 0;
      for (int s = t.first_step; s <= t.last_step; ++s) {
        bool fixed = false;
        for (int f = 0; f < t.n_fixed_steps; ++f) fixed |= (t.fixed_steps[f] == s);
        steps += !fixed;
      }
      L.n_coll_cand += steps * d.robot.n_spheres * d.n_obstacles;
    }
  }
  L.cart_stride = has_vel ? 2 * D : D;
  L.coll_stride = has_cast ? 2 * D + 3 : D + 3;
  return L;
}
void putResults(const TrajProblem& tp, const BasicTrustRegionSQP& opt, int b, tb200_results* out) {
  const OptResults& r = opt.results();
  const size_t N = r.x.size(), nc = tp.cost_names.size(), nk = tp.cnt_names.size();
  if (out->x) std::memcpy(out->x + b * N, r.x.data(), sizeof(double) * N);
  if (out->status) out->status[b] = r.status;
  if (out->total_cost) out->total_cost[b] = r.total_cost;
  if (out->cost_vals)
    for (size_t i = 0; i < nc; ++i) out->cost_vals[b * nc + i] = r.cost_vals[i];
  if (out->cnt_viols)
    for (size_t i = 0; i < nk; ++i) out->cnt_viols[b * nk + i] = r.cnt_viols[i];
  if (out->n_qp_solves) out->n_qp_solves[b] = r.n_qp_solves;
  if (out->n_func_evals) out->n_func_evals[b] = r.n_func_evals;
  if (out->n_admm_iters) out->n_admm_iters[b] = static_cast<int>(tp.prob->model()->totalAdmmIters());
}

// The iteration log of every trajectory, [B][cap][...] (record k of trajectory b at b * cap + k); any array may be NULL.
struct oracle_records {
  int cap;
  int32_t* n;                // [B] records written (at most cap)
  double* trace;             // [B][cap][14] the TraceEntry columns of the record's QP solve; NaN for record 0
  double* merit_coeffs;      // [B][cap][n_cnts]
  double* model_cost_vals;   // [B][cap][n_costs]
  double* model_cnt_viols;   // [B][cap][n_cnts]
  double* cost_vals;         // [B][cap][n_costs]
  double* cnt_viols;         // [B][cap][n_cnts]
  double* x;                 // [B][cap][T * D]
};
// one TraceEntry as 14 doubles
void traceRow(const TraceEntry& te, double* o) {
  o[0] = te.merit_round; o[1] = te.iter; o[2] = te.trust; o[3] = te.old_merit; o[4] = te.model_merit;
  o[5] = te.new_merit; o[6] = te.qp_status; o[7] = te.admm_iters; o[8] = te.action;
  o[9] = te.pri; o[10] = te.dua; o[11] = te.rho; o[12] = te.polish; o[13] = te.warm;
}
void putRecords(const BasicTrustRegionSQP& opt, int b, const oracle_records& rec) {
  auto put = [](double* dst, size_t at, const Vec& v) {
    if (dst) std::memcpy(dst + at * v.size(), v.data(), sizeof(double) * v.size());
  };
  const size_t n = std::min(opt.records.size(), static_cast<size_t>(rec.cap));
  if (rec.n) rec.n[b] = static_cast<int32_t>(n);
  for (size_t k = 0; k < n; ++k) {
    const size_t at = static_cast<size_t>(b) * rec.cap + k;
    if (rec.trace) {
      double* o = rec.trace + at * 14;
      if (k == 0)
        std::fill(o, o + 14, std::numeric_limits<double>::quiet_NaN());
      else
        traceRow(opt.trace[k - 1], o);
    }
    const IterRecord& r = opt.records[k];
    put(rec.merit_coeffs, at, r.merit_coeffs);
    put(rec.model_cost_vals, at, r.model_cost_vals);
    put(rec.model_cnt_viols, at, r.model_cnt_viols);
    put(rec.cost_vals, at, r.cost_vals);
    put(rec.cnt_viols, at, r.cnt_viols);
    put(rec.x, at, r.x);
  }
}

// BasicTrustRegionSQP::optimize() for trajectories [b0, b1) of the batch, OpenMP over trajectories: setup(opt, b)
// configures a trajectory's driver, collect(opt, b) copies out what the entry point returns beyond the results.
template <class Setup, class Collect>
int solveBatch(const tb200_problem_desc* desc, int b0, int b1, int n_threads, tb200_results* out, double* seconds,
               Setup setup, Collect collect) {
  int err = 0;
  const int cast_cap = tb200inl_cast_rows_per_pair(desc);
  const auto t0 = std::chrono::steady_clock::now();
#ifdef _OPENMP
  if (n_threads > 0) omp_set_num_threads(n_threads);
#endif
#pragma omp parallel for schedule(dynamic)
  for (int b = b0; b < b1; ++b) {
    try {
      TrajProblem tp = buildProblem(*desc, b, cast_cap);
      BasicTrustRegionSQP opt(tp.prob);
      opt.params() = sqpParamsFrom(desc->sqp);
      setup(opt, b);
      opt.initialize(tp.init);
      opt.optimize();
      putResults(tp, opt, b, out);
      collect(opt, b);
    } catch (const std::exception& e) {
#pragma omp critical
      {
        g_err = e.what();
        err = 1;
      }
    }
  }
  if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return err;
}
}  // namespace

extern "C" {

const char* oracle_last_error() { return g_err.c_str(); }

int oracle_layout(const tb200_problem_desc* desc, tb200_layout* out) {
  try {
    TrajProblem tp = buildProblem(*desc, 0);
    Layout L = layoutOf(*desc, tp);
    out->n_costs = L.n_costs;
    out->n_cnts = L.n_cnts;
    out->n_cart_rows = L.n_cart_rows;
    out->cart_jac_stride = L.cart_stride;
    out->n_coll_cand = L.n_coll_cand;
    out->coll_row_stride = L.coll_stride;
    out->n_vars = desc->n_steps * desc->robot.n_dof;
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// BasicTrustRegionSQP::optimize() for trajectories [b0, b1) of the batch, OpenMP over trajectories; desc->sqp.max_time
// is not read.  seconds: NULL or the wall time of the whole call.
// trace_*: optional decision trace of trajectory `trace_b` (max trace_cap entries of 14 doubles).
int oracle_solve_batch(const tb200_problem_desc* desc, int b0, int b1, int n_threads, tb200_results* out,
                       double* seconds, int trace_b, double* trace_out, int trace_cap, int* trace_len) {
  return solveBatch(desc, b0, b1, n_threads, out, seconds, [](BasicTrustRegionSQP&, int) {},
                    [&](const BasicTrustRegionSQP& opt, int b) {
                      if (b != trace_b || !trace_out) return;
                      const int n = std::min(static_cast<int>(opt.trace.size()), trace_cap);
                      for (int k = 0; k < n; ++k) traceRow(opt.trace[k], trace_out + k * 14);
                      if (trace_len) *trace_len = n;
                    });
}

// oracle_solve_batch with a stop rule and the iteration log.
// stop_rule: 0 none (desc->sqp.max_time is not read), 1 a wall clock per trajectory against desc->sqp.max_time,
// 2 the QP budget qp_budget[b] ([B]).  ended: [B] or NULL, 1 where the stop rule ended the trajectory.
// records: NULL, or the iteration log of every trajectory.
int oracle_solve_batch_ext(const tb200_problem_desc* desc, int b0, int b1, int n_threads, int stop_rule,
                           const int32_t* qp_budget, tb200_results* out, int32_t* ended, const oracle_records* records,
                           double* seconds) {
  return solveBatch(
      desc, b0, b1, n_threads, out, seconds,
      [&](BasicTrustRegionSQP& opt, int b) {
        opt.setStopRule(static_cast<BasicTrustRegionSQP::StopRule>(stop_rule), desc->sqp.max_time,
                        qp_budget ? qp_budget[b] : 0);
        opt.record = records != nullptr;
      },
      [&](const BasicTrustRegionSQP& opt, int b) {
        if (ended) ended[b] = opt.ended ? 1 : 0;
        if (records) putRecords(opt, b, *records);
      });
}

// costs[i]->convex/value and cnts[i]->convex/violation at x for trajectories [b0,b1), written in the
// fixed dense layout of tb200_convexify_out.
int oracle_convexify_batch(const tb200_problem_desc* desc, int b0, int b1, const double* x, tb200_convexify_out* out) {
  const int T = desc->n_steps, D = desc->robot.n_dof;
  const int cast_cap = tb200inl_cast_rows_per_pair(desc);
  try {
    for (int b = b0; b < b1; ++b) {
      TrajProblem tp = buildProblem(*desc, b, cast_cap);
      const Layout L = layoutOf(*desc, tp);
      Vec xv(x + static_cast<size_t>(b) * T * D, x + static_cast<size_t>(b + 1) * T * D);
      if (out->cart_err || out->cart_jac) {
        Vec err;
        std::vector<Vec> jac;
        for (auto& h : tp.cart_hooks) h(xv, err, jac);
        for (int r = 0; r < L.n_cart_rows; ++r) {
          if (out->cart_err) out->cart_err[static_cast<size_t>(b) * L.n_cart_rows + r] = err[r];
          if (out->cart_jac) {
            double* o = out->cart_jac + (static_cast<size_t>(b) * L.n_cart_rows + r) * L.cart_stride;
            for (int j = 0; j < L.cart_stride; ++j) o[j] = j < static_cast<int>(jac[r].size()) ? jac[r][j] : 0.0;
          }
        }
      }
      if (out->coll_rows) {
        std::vector<Vec> rows;
        for (auto& h : tp.coll_hooks) h(xv, rows);
        for (int r = 0; r < L.n_coll_cand; ++r)
          std::memcpy(out->coll_rows + (static_cast<size_t>(b) * L.n_coll_cand + r) * L.coll_stride, rows[r].data(),
                      sizeof(double) * L.coll_stride);
      }
      if (out->cost_vals) {
        const auto& costs = tp.prob->getCosts();
        for (size_t i = 0; i < costs.size(); ++i) out->cost_vals[b * costs.size() + i] = costs[i]->value(xv);
      }
      if (out->cnt_viols) {
        const auto cnts = tp.prob->getConstraints();
        for (size_t i = 0; i < cnts.size(); ++i) out->cnt_viols[b * cnts.size() + i] = cnts[i]->violation(xv);
      }
    }
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// One Model::optimize() on the QP convexified at x (optimizers.cpp:781-814 for a single try).
// Also returns the KKT residuals of the returned (x,y) on the unscaled QP.
int oracle_qp_solve_batch(const tb200_problem_desc* desc, int b0, int b1, const double* x, const double* trust,
                          const double* merit_coeffs, double* new_x, int32_t* qp_status, double* model_cost_vals,
                          double* model_cnt_viols, int32_t* admm_iters, double* kkt /*[B][3]*/,
                          int32_t* polish /*[B]*/) {
  const int T = desc->n_steps, D = desc->robot.n_dof, N = T * D;
  const int cast_cap = tb200inl_cast_rows_per_pair(desc);
  try {
    for (int b = b0; b < b1; ++b) {
      TrajProblem tp = buildProblem(*desc, b, cast_cap);
      Model* model = tp.prob->model();
      const size_t nc = tp.cost_names.size(), nk = tp.cnt_names.size();
      Vec xv(x + static_cast<size_t>(b) * N, x + static_cast<size_t>(b + 1) * N);
      const ConvexModels cm = convexifyProblem(*tp.prob, xv, merit_coeffs + b * nk);
      setTrustBoxConstraints(*tp.prob, xv, trust[b]);
      const CvxStatus st = model->optimize();
      const Vec& sol = model->solution();
      Vec mc, mk;
      cm.values(sol.data(), mc, mk);
      if (new_x) std::memcpy(new_x + static_cast<size_t>(b) * N, sol.data(), sizeof(double) * N);
      if (qp_status) qp_status[b] = st;
      if (model_cost_vals) std::copy(mc.begin(), mc.end(), model_cost_vals + b * nc);
      if (model_cnt_viols) std::copy(mk.begin(), mk.end(), model_cnt_viols + b * nk);
      if (admm_iters) admm_iters[b] = model->lastResult().iters;
      if (polish) polish[b] = model->lastResult().polish;
      if (kkt) {
        QP qp;
        model->buildQP(qp);
        qp_kkt_residuals(qp, model->lastResult().x, model->lastResult().y, kkt[b * 3], kkt[b * 3 + 1], kkt[b * 3 + 2]);
      }
    }
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// ---- kinematics probes (pinning FK / transform error against closed forms in the tests)
int oracle_fk(const tb200_robot* robot, const double* q, double* frames /*[n_segments][12] R row-major + p*/) {
  Robot r(*robot);
  std::vector<Pose> fr;
  r.fk(q, fr);
  for (size_t s = 0; s < fr.size(); ++s) {
    std::memcpy(frames + s * 12, fr[s].R, sizeof(double) * 9);
    std::memcpy(frames + s * 12 + 9, fr[s].p, sizeof(double) * 3);
  }
  return 0;
}
int oracle_jacobian(const tb200_robot* robot, const double* q, int link, const double* point /*NULL = link origin*/,
                    double* J /*[6][n_dof]*/) {
  Robot r(*robot);
  std::vector<Pose> fr;
  r.fk(q, fr);
  std::vector<Vec> Jv;
  r.jacobian(fr, link, point ? point : fr[link].p, Jv);
  for (int i = 0; i < 6; ++i) std::memcpy(J + i * r.n_dof, Jv[i].data(), sizeof(double) * r.n_dof);
  return 0;
}
// avoid_singularity probes: sigma, u[6], v[D] of a 6 x D matrix (row-major); the Jacobian, sigma, err and the unscaled
// gradient of one waypoint (any output may be NULL)
int oracle_sing_svd_min(const double* J, int D, double* sigma, double* u, double* v) {
  sing::jacobiSvdMin(J, D, *sigma, u, v);
  return 0;
}
int oracle_sing_err_grad(const tb200_robot* robot, const double* q, int link, double lambda, double* J, double* sigma,
                         double* err, double* grad) {
  try {
    Robot r(*robot);
    std::vector<double> Jv;
    sing::jacobianAt(r, q, link, Jv);
    if (J) std::memcpy(J, Jv.data(), sizeof(double) * Jv.size());
    sing::errGrad(r, q, link, lambda, err, grad, sigma);
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// (term, step) of every object in OptProb order (the costs, then the EQ and the INEQ constraints), as
// tb200_problem_objects lists them; term and step: [n_costs + n_cnts]
int oracle_objects(const tb200_problem_desc* desc, int32_t* term, int32_t* step) {
  try {
    TrajProblem tp = buildProblem(*desc, 0);
    int n = 0;
    for (const auto& c : tp.prob->getCosts()) {
      term[n] = c->term;
      step[n++] = c->step;
    }
    for (const auto& c : tp.prob->getConstraints()) {
      term[n] = c->term;
      step[n++] = c->step;
    }
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

void oracle_transform_error(const double* t1 /*xyz+wxyz*/, const double* t2, double* err6) {
  calcTransformError(poseFromXyzWxyz(t1, t1 + 3), poseFromXyzWxyz(t2, t2 + 3), err6);
}

// ---- expression / canonical-form probes (reference known-answers: solver-utils-unit.cpp)
// quadratic of (coeffs . x + constant)^2 -> dense Q, q, nnz
int oracle_square_to_dense(const double* coeffs, int n, double constant, int halved, int force_diag, double* Q,
                           double* q, int* nnz) {
  AffExpr a;
  a.constant = constant;
  for (int i = 0; i < n; ++i) {
    a.vars.push_back(i);
    a.coeffs.push_back(coeffs[i]);
  }
  QuadExpr sq = exprSquare(a);
  Vec Qv, qv;
  quadToDense(sq, n, halved != 0, force_diag != 0, Qv, qv, *nnz);
  std::memcpy(Q, Qv.data(), sizeof(double) * n * n);
  std::memcpy(q, qv.data(), sizeof(double) * n);
  return 0;
}
// affine row -> (A row, u) of the Model canonical form
int oracle_aff_to_row(const double* coeffs, int n, double constant, double* row, double* u) {
  AffExpr a;
  a.constant = constant;
  for (int i = 0; i < n; ++i) {
    a.vars.push_back(i);
    a.coeffs.push_back(coeffs[i]);
  }
  Model m;
  for (int i = 0; i < n; ++i) m.addVar();
  m.addIneqCnt(a);
  QP qp;
  m.buildQP(qp);
  std::fill(row, row + n, 0.0);
  for (int k = qp.A.ptr[0]; k < qp.A.ptr[1]; ++k) row[qp.A.idx[k]] = qp.A.val[k];
  *u = qp.u[0];
  return 0;
}
int oracle_dense_to_csc(const double* M, int rows, int cols, int upper_only, long long* row_idx, long long* col_ptr,
                        double* data, int* nnz) {
  std::vector<long long> ri, cp;
  Vec d;
  denseToCsc(Vec(M, M + rows * cols), rows, cols, upper_only != 0, ri, cp, d);
  std::copy(ri.begin(), ri.end(), row_idx);
  std::copy(cp.begin(), cp.end(), col_ptr);
  std::copy(d.begin(), d.end(), data);
  *nnz = static_cast<int>(d.size());
  return 0;
}
// objective value probes of solver-interface-unit.cpp:136-237: (a1 x0 + c1)(a2 x1 + c2) style products are
// built there with exprMult; here the equivalent QuadExpr is evaluated through QuadExpr::value.
double oracle_quad_value(const double* aff_coeffs, int n, double constant, const int* v1, const int* v2,
                         const double* qc, int nq, const double* x) {
  QuadExpr q;
  q.aff.constant = constant;
  for (int i = 0; i < n; ++i) {
    q.aff.vars.push_back(i);
    q.aff.coeffs.push_back(aff_coeffs[i]);
  }
  for (int k = 0; k < nq; ++k) {
    q.v1.push_back(v1[k]);
    q.v2.push_back(v2[k]);
    q.coeffs.push_back(qc[k]);
  }
  return q.value(x);
}

// Generic small QP through the OSQP-equivalent solver (dense inputs), for KKT / known-answer tests.
int oracle_qp_dense(int n, int m, const double* P /*n*n symmetric*/, const double* q, const double* A /*m*n*/,
                    const double* l, const double* u, const tb200_qp_settings* st, double* x, double* y, int* status,
                    int* iters, int* polish) {
  QP qp;
  qp.n = n;
  qp.m = m;
  qp.Pu.cols = n;
  for (int i = 0; i < n; ++i) {
    std::vector<int> c;
    Vec v;
    for (int j = i; j < n; ++j)
      if (P[i * n + j] != 0.0) {
        c.push_back(j);
        v.push_back(P[i * n + j]);
      }
    qp.Pu.addRow(c, v);
  }
  qp.q.assign(q, q + n);
  qp.A.cols = n;
  for (int r = 0; r < m; ++r) {
    std::vector<int> c;
    Vec v;
    for (int j = 0; j < n; ++j)
      if (A[r * n + j] != 0.0) {
        c.push_back(j);
        v.push_back(A[r * n + j]);
      }
    qp.A.addRow(c, v);
  }
  qp.l.assign(l, l + m);
  qp.u.assign(u, u + m);
  QPResult r = qp_solve(qp, st ? qpSettingsFrom(*st) : QPSettings(), nullptr);
  std::copy(r.x.begin(), r.x.end(), x);
  std::copy(r.y.begin(), r.y.end(), y);
  *status = r.status;
  *iters = r.iters;
  *polish = r.polish;
  return 0;
}

// ---- the reference's toy NLPs (trajopt_sco/test/small-problems-unit.cpp:48-172)
static double sq(double v) { return v * v; }
int oracle_small_problem(int id, double* x_out, int* status, int* n_out) {
  auto prob = std::make_shared<OptProb>();
  SQPParams p;
  Vec init;
  ScalarFn f;
  VectorFn g;
  CntType ct = INEQ;
  bool full_hess = true, has_g = true;
  switch (id) {
    case 0:  // QuadraticSeparable
      f = [](const Vec& x) { return x[0] * x[0] + sq(x[1] - 1) + sq(x[2] - 2); };
      init = {3, 4, 5};
      p.trust_box_size = 100;
      full_hess = false;
      has_g = false;
      break;
    case 1:  // QuadraticNonseparable
      f = [](const Vec& x) { return sq(x[0] - x[1] + 3 * x[2]) + sq(x[0] - 1) + sq(x[2] - 2); };
      init = {3, 4, 5};
      p.trust_box_size = 100;
      p.min_trust_box_size = 1e-5;
      p.min_approx_improve = 1e-6;
      has_g = false;
      break;
    case 2:  // TP1
      f = [](const Vec& x) { return 1 * sq(x[1] - sq(x[0])) + sq(1 - x[0]); };
      g = [](const Vec& x) { return Vec{-1.5 - x[1]}; };
      init = {-2, 1};
      break;
    case 3:  // TP3
      f = [](const Vec& x) { return x[1] + 1e-5 * sq(x[1] - x[0]); };
      g = [](const Vec& x) { return Vec{0 - x[1]}; };
      init = {10, 1};
      break;
    case 4:  // TP6
      f = [](const Vec& x) { return sq(1 - x[0]); };
      g = [](const Vec& x) { return Vec{10 * (x[1] - sq(x[0]))}; };
      ct = EQ;
      init = {10, 1};
      break;
    case 5:  // TP7
      f = [](const Vec& x) { return std::log(1 + sq(x[0])) - x[1]; };
      g = [](const Vec& x) { return Vec{sq(1 + sq(x[0])) + sq(x[1]) - 4}; };
      ct = EQ;
      init = {2, 2};
      break;
    default:
      return 1;
  }
  const int n = static_cast<int>(init.size());
  std::vector<int> vars = prob->createVariables(n);
  prob->addCost(std::make_shared<CostFromFunc>(f, vars, full_hess));
  if (has_g) {
    prob->addConstraint(std::make_shared<ConstraintFromErrFunc>(g, MatrixFn(), vars, Vec(), ct));
    p.max_iter = 1000;
    p.min_trust_box_size = 1e-5;
    p.min_approx_improve = 1e-10;
    p.initial_merit_error_coeff = 1;
  }
  BasicTrustRegionSQP opt(prob);
  opt.params() = p;
  opt.initialize(init);
  *status = opt.optimize();
  for (int i = 0; i < n; ++i) x_out[i] = opt.results().x[i];
  *n_out = n;
  return 0;
}

// the trust box of one variable (setTrustBoxConstraints, optimizers.cpp:151-170)
int oracle_trust_box(double x, double lb, double ub, double trust, double* lo, double* hi) {
  trustBox(x, lb, ub, trust, *lo, *hi);
  return 0;
}

int oracle_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
}
