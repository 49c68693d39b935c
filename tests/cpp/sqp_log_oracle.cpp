// CPU model of the SQP iteration log (DESIGN.md section 4.7), for tests/test_sqp_log.py.  It is the oracle's SQP driver
// (oracle/sco.cpp, BasicTrustRegionSQP::optimize) with full records, built on the oracle's public pieces and linked
// against liboracle.so; the oracle's own driver, the yardstick of every solve, is left as it is.
//
// Records as the device writes them: record 0 the state after the first evaluation (clamped start, its exact values,
// the initial merit coefficients), then one per QP solve, failed ones included: the oracle's 14 TraceEntry columns
// (round, iter, trust, old / model / new merit, QP status, ADMM iterations, action, residuals, rho, polish, warm), the
// merit coefficients in force, the model value of every object at the QP solution, the exact values there and the
// point.  A failed QP has no model, values or point: NaN (its trace row holds zero merits, as the oracle's does).
#include <algorithm>
#include <cstring>
#include <limits>
#include <string>

#include "trajopt.hpp"

using namespace oracle;

namespace {
thread_local std::string g_err;

double vecSum(const Vec& v) {
  double s = 0;
  for (double e : v) s += e;
  return s;
}
double vecDot(const Vec& a, const Vec& b) {
  double s = 0;
  for (size_t i = 0; i < a.size(); ++i) s += a[i] * b[i];
  return s;
}
double vecMax(const Vec& v) { return *std::max_element(v.begin(), v.end()); }

struct Record {
  double trace[14];
  Vec mu, mc, mk, vc, vk, x;
};

OptResults optimizeLogged(OptProb& prob, SQPParams param, const Vec& x0, std::vector<Record>& log) {
  Model* model = prob.model();
  const auto constraints = prob.getConstraints();
  const auto& costs = prob.getCosts();
  const double nan = std::numeric_limits<double>::quiet_NaN();
  Vec merit_error_coeffs(constraints.size(), param.initial_merit_error_coeff);
  OptResults res;
  res.x = prob.getClosestFeasiblePoint(x0);
  OptStatus retval = OPT_INVALID;
  auto evalCosts = [&](const Vec& x) {
    Vec out(costs.size());
    for (size_t i = 0; i < costs.size(); ++i) out[i] = costs[i]->value(x);
    return out;
  };
  auto evalViols = [&](const Vec& x) {
    Vec out(constraints.size());
    for (size_t i = 0; i < constraints.size(); ++i) out[i] = constraints[i]->violation(x);
    return out;
  };
  auto trustBoxes = [&](const Vec& x) {
    for (size_t i = 0; i < x.size(); ++i) {
      double lo, hi;
      trustBox(x[i], prob.lower()[i], prob.upper()[i], param.trust_box_size, lo, hi);
      model->setVarBounds(static_cast<int>(i), lo, hi);
    }
  };
  auto failed = [&](size_t n) { return Vec(n, nan); };

  for (int merit_increases = 0; merit_increases < param.max_merit_coeff_increases; ++merit_increases) {
    for (int iter = 1;; ++iter) {
      if (res.cost_vals.empty() && res.cnt_viols.empty()) {  // first iteration only
        res.cnt_viols = evalViols(res.x);
        res.cost_vals = evalCosts(res.x);
        ++res.n_func_evals;
        Record r0;
        std::fill(r0.trace, r0.trace + 14, nan);
        r0.mu = merit_error_coeffs;
        r0.mc = failed(costs.size());
        r0.mk = failed(constraints.size());
        r0.vc = res.cost_vals;
        r0.vk = res.cnt_viols;
        r0.x = res.x;
        log.push_back(r0);
      }
      model->truncateToPermanent();
      std::vector<std::shared_ptr<ConvexObjective>> cost_models, cnt_cost_models;
      std::vector<std::shared_ptr<ConvexConstraints>> cnt_models;
      for (auto& c : costs) cost_models.push_back(c->convex(res.x, model));
      for (auto& c : constraints) cnt_models.push_back(c->convex(res.x, model));
      for (size_t c = 0; c < cnt_models.size(); ++c) {
        auto obj = std::make_shared<ConvexObjective>(model);
        for (const AffExpr& a : cnt_models[c]->eqs) obj->addAbs(a, merit_error_coeffs[c]);
        for (const AffExpr& a : cnt_models[c]->ineqs) obj->addHinge(a, merit_error_coeffs[c]);
        cnt_cost_models.push_back(obj);
      }
      for (auto& c : cost_models) c->addConstraintsToModel();
      for (auto& c : cnt_cost_models) c->addConstraintsToModel();
      QuadExpr objective;
      for (auto& c : cost_models) exprInc(objective, c->quad);
      for (auto& c : cnt_cost_models) exprInc(objective, c->quad);
      model->setObjective(objective);

      int qp_solver_failures = 0;
      bool converged = false;
      while (param.trust_box_size >= param.min_trust_box_size) {
        trustBoxes(res.x);
        const CvxStatus status = model->optimize();
        ++res.n_qp_solves;
        const QPResult& q = model->lastResult();
        Record rec;
        const double tr[14] = {double(merit_increases), double(iter), param.trust_box_size, 0, 0, 0, double(q.status),
                               double(q.iters), 3, q.admm_pri, q.admm_dua, q.rho, double(q.polish), double(q.warm)};
        std::copy(tr, tr + 14, rec.trace);
        rec.mu = merit_error_coeffs;
        if (status != CVX_SOLVED) {
          rec.trace[9] = rec.trace[10] = rec.trace[11] = rec.trace[12] = rec.trace[13] = 0;  // (TraceEntry defaults)
          rec.mc = failed(costs.size()); rec.mk = failed(constraints.size());
          rec.vc = failed(costs.size()); rec.vk = failed(constraints.size()); rec.x = failed(res.x.size());
          log.push_back(rec);
          if (qp_solver_failures < (param.max_qp_solver_failures - 1)) {
            param.trust_box_size *= param.trust_shrink_ratio;
            qp_solver_failures++;
            continue;
          }
          if (qp_solver_failures == (param.max_qp_solver_failures - 1)) {
            param.trust_box_size = param.min_trust_box_size;
            qp_solver_failures++;
            continue;
          }
          retval = OPT_FAILED;
          goto cleanup;
        }
        const Vec& mv = model->solution();
        Vec model_cost_vals(cost_models.size()), model_cnt_viols(cnt_models.size());
        for (size_t i = 0; i < cost_models.size(); ++i) model_cost_vals[i] = cost_models[i]->value(mv.data());
        for (size_t i = 0; i < cnt_models.size(); ++i) model_cnt_viols[i] = cnt_models[i]->violation(mv.data());
        Vec new_x(mv.begin(), mv.begin() + static_cast<long>(res.x.size()));
        const Vec new_cost_vals = evalCosts(new_x);
        const Vec new_cnt_viols = evalViols(new_x);
        const double old_merit = vecSum(res.cost_vals) + vecDot(res.cnt_viols, merit_error_coeffs);
        const double model_merit = vecSum(model_cost_vals) + vecDot(model_cnt_viols, merit_error_coeffs);
        const double new_merit = vecSum(new_cost_vals) + vecDot(new_cnt_viols, merit_error_coeffs);
        const double approx_merit_improve = old_merit - model_merit;
        const double exact_merit_improve = old_merit - new_merit;
        const double merit_improve_ratio = exact_merit_improve / approx_merit_improve;
        ++res.n_func_evals;
        rec.trace[3] = old_merit; rec.trace[4] = model_merit; rec.trace[5] = new_merit;
        rec.mc = model_cost_vals; rec.mk = model_cnt_viols; rec.vc = new_cost_vals; rec.vk = new_cnt_viols; rec.x = new_x;
        if (approx_merit_improve < param.min_approx_improve ||
            approx_merit_improve / old_merit < param.min_approx_improve_frac) {
          rec.trace[8] = 2;
          log.push_back(rec);
          converged = true;
          break;
        } else if (exact_merit_improve < 0 || merit_improve_ratio < param.improve_ratio_threshold) {
          rec.trace[8] = 0;
          log.push_back(rec);
          param.trust_box_size *= param.trust_shrink_ratio;
        } else {
          rec.trace[8] = 1;
          log.push_back(rec);
          res.x = new_x;
          res.cost_vals = new_cost_vals;
          res.cnt_viols = new_cnt_viols;
          param.trust_box_size *= param.trust_expand_ratio;
          break;
        }
      }
      if (converged || param.trust_box_size < param.min_trust_box_size) goto penaltyadjustment;
      if (iter >= param.max_iter) {
        retval = OPT_SCO_ITERATION_LIMIT;
        if (res.cnt_viols.empty() || vecMax(res.cnt_viols) < param.cnt_tolerance) retval = OPT_CONVERGED;
        goto cleanup;
      }
    }
  penaltyadjustment:
    if (res.cnt_viols.empty() || vecMax(res.cnt_viols) < param.cnt_tolerance) {
      retval = OPT_CONVERGED;
      goto cleanup;
    }
    if (param.inflate_constraints_individually) {
      for (size_t i = 0; i < res.cnt_viols.size(); ++i)
        if (res.cnt_viols[i] > param.cnt_tolerance) merit_error_coeffs[i] *= param.merit_coeff_increase_ratio;
    } else {
      for (double& c : merit_error_coeffs) c *= param.merit_coeff_increase_ratio;
    }
    param.trust_box_size = std::fmax(param.trust_box_size, param.min_trust_box_size / param.trust_shrink_ratio * 1.5);
  }
  retval = OPT_PENALTY_ITERATION_LIMIT;
cleanup:
  res.status = retval;
  res.total_cost = vecSum(res.cost_vals);
  return res;
}

void put(double* dst, size_t b, size_t cap, size_t r, const Vec& v) {
  if (dst) std::memcpy(dst + (b * cap + r) * v.size(), v.data(), sizeof(double) * v.size());
}
}  // namespace

extern "C" {

const char* slo_last_error() { return g_err.c_str(); }

// Trajectories [b0, b1) of the batch, OpenMP over trajectories; up to cap records each (n_records[b] of them, the rest
// untouched).  trace [B][cap][14]; mu, model_cnt_viols, new_cnt_viols [B][cap][n_cnts]; model_cost_vals, new_cost_vals
// [B][cap][n_costs]; x [B][cap][T*D].  Any array may be NULL.
int slo_solve_batch(const tb200_problem_desc* desc, int b0, int b1, int cap, tb200_results* out, int* n_records,
                    double* trace, double* mu, double* model_cost_vals, double* model_cnt_viols, double* new_cost_vals,
                    double* new_cnt_viols, double* x) {
  const int T = desc->n_steps, D = desc->robot.n_dof;
  const int cast_cap = tb200inl_cast_rows_per_pair(desc);
  int err = 0;
#pragma omp parallel for schedule(dynamic)
  for (int b = b0; b < b1; ++b) {
    try {
      TrajProblem tp = buildProblem(*desc, b, cast_cap);
      std::vector<Record> log;
      const OptResults r = optimizeLogged(*tp.prob, sqpParamsFrom(desc->sqp), tp.init, log);
      const size_t nc = tp.cost_names.size(), nk = tp.cnt_names.size();
      if (out->x) std::memcpy(out->x + static_cast<size_t>(b) * T * D, r.x.data(), sizeof(double) * T * D);
      if (out->status) out->status[b] = r.status;
      if (out->total_cost) out->total_cost[b] = r.total_cost;
      if (out->cost_vals)
        for (size_t i = 0; i < nc; ++i) out->cost_vals[b * nc + i] = r.cost_vals[i];
      if (out->cnt_viols)
        for (size_t i = 0; i < nk; ++i) out->cnt_viols[b * nk + i] = r.cnt_viols[i];
      if (out->n_qp_solves) out->n_qp_solves[b] = r.n_qp_solves;
      if (out->n_func_evals) out->n_func_evals[b] = r.n_func_evals;
      if (out->n_admm_iters) out->n_admm_iters[b] = static_cast<int>(tp.prob->model()->totalAdmmIters());
      const size_t n = std::min(log.size(), static_cast<size_t>(cap));
      if (n_records) n_records[b] = static_cast<int>(n);
      for (size_t k = 0; k < n; ++k) {
        if (trace) std::memcpy(trace + (b * static_cast<size_t>(cap) + k) * 14, log[k].trace, sizeof(double) * 14);
        put(mu, b, cap, k, log[k].mu);
        put(model_cost_vals, b, cap, k, log[k].mc);
        put(model_cnt_viols, b, cap, k, log[k].mk);
        put(new_cost_vals, b, cap, k, log[k].vc);
        put(new_cnt_viols, b, cap, k, log[k].vk);
        put(x, b, cap, k, log[k].x);
      }
    } catch (const std::exception& ex) {
#pragma omp critical
      {
        g_err = ex.what();
        err = 1;
      }
    }
  }
  return err;
}

}  // extern "C"
