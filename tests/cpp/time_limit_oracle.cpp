// CPU model of the SQP time limit (sco::BasicTrustRegionSQPParameters::max_time, optimizers.cpp:738-753), for
// tests/test_time_limit.py.  It is the oracle's SQP driver (oracle/sco.cpp, BasicTrustRegionSQP::optimize) with the
// check added, built on the oracle's public pieces and linked against liboracle.so; the oracle's own driver, the
// yardstick of every untimed solve, is left as it is.
//
// The check sits where the reference has it and where the device makes it (DESIGN.md section 6): at the top of every
// SQP iteration (iter = 1 of each merit round and every ++iter), never on a trust-region or QP-failure retry, and
// first after the initial evaluation.  A trajectory stopped there keeps its accepted x, cost_vals and cnt_viols;
// its status is OPT_CONVERGED when it has no constraints or max(cnt_viols) < cnt_tolerance, else OPT_TIME_LIMIT.
//
// Two clocks:
//   * qp_budget == NULL: wall time, one std::chrono::steady_clock per trajectory started in optimize(), against
//     desc->sqp.max_time (the reference's clock model);
//   * qp_budget != NULL: a deterministic stand-in, "stop at the first iteration top with n_qp_solves >= qp_budget[b]",
//     which reproduces a time-limited device run exactly once the device's QP counts are known.
#include <algorithm>
#include <chrono>
#include <cstring>
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

// oracle/sco.cpp BasicTrustRegionSQP::optimize() plus the time-limit check; `ended` = stopped by the check.
OptResults optimizeTimed(OptProb& prob, SQPParams param, double max_time, const Vec& x0, const int* qp_budget, bool& ended) {
  Model* model = prob.model();
  const auto constraints = prob.getConstraints();
  const auto& costs = prob.getCosts();
  Vec merit_error_coeffs(constraints.size(), param.initial_merit_error_coeff);
  OptResults res;
  res.x = prob.getClosestFeasiblePoint(x0);
  OptStatus retval = OPT_INVALID;
  ended = false;
  const auto start = std::chrono::steady_clock::now();
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

  for (int merit_increases = 0; merit_increases < param.max_merit_coeff_increases; ++merit_increases) {
    for (int iter = 1;; ++iter) {
      if (res.cost_vals.empty() && res.cnt_viols.empty()) {  // first iteration only
        res.cnt_viols = evalViols(res.x);
        res.cost_vals = evalCosts(res.x);
        ++res.n_func_evals;
      }
      const bool over = qp_budget ? res.n_qp_solves >= *qp_budget
                                  : std::chrono::duration<double>(std::chrono::steady_clock::now() - start).count() >
                                        max_time;
      if (over) {
        ended = true;
        retval = (res.cnt_viols.empty() || vecMax(res.cnt_viols) < param.cnt_tolerance) ? OPT_CONVERGED : OPT_TIME_LIMIT;
        goto cleanup;
      }
      model->truncateToPermanent();
      {
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
          if (status != CVX_SOLVED) {
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
          if (approx_merit_improve < param.min_approx_improve ||
              approx_merit_improve / old_merit < param.min_approx_improve_frac) {
            converged = true;
            break;
          } else if (exact_merit_improve < 0 || merit_improve_ratio < param.improve_ratio_threshold) {
            param.trust_box_size *= param.trust_shrink_ratio;
          } else {
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
}  // namespace

extern "C" {

const char* tl_oracle_last_error() { return g_err.c_str(); }

// Trajectories [b0, b1) of the batch, OpenMP over trajectories.  qp_budget: [B] or NULL (wall clock, desc->sqp.max_time).
// ended: [B] or NULL, 1 where the time limit ended the trajectory.
int tl_oracle_solve_batch(const tb200_problem_desc* desc, int b0, int b1, const int* qp_budget, tb200_results* out,
                          int* ended) {
  const int T = desc->n_steps, D = desc->robot.n_dof;
  const int cast_cap = tb200inl_cast_rows_per_pair(desc);
  int err = 0;
#pragma omp parallel for schedule(dynamic)
  for (int b = b0; b < b1; ++b) {
    try {
      TrajProblem tp = buildProblem(*desc, b, cast_cap);
      SQPParams param = sqpParamsFrom(desc->sqp);
      bool e = false;
      const OptResults r = optimizeTimed(*tp.prob, param, desc->sqp.max_time, tp.init, qp_budget ? qp_budget + b : nullptr, e);
      const size_t nc = tp.cost_names.size(), nk = tp.cnt_names.size();
      if (ended) ended[b] = e ? 1 : 0;
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
