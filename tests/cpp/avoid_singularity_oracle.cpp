// CPU model of the avoid_singularity term (AvoidSingularityTermInfo, trajopt/src/kinematic_terms.cpp:586-642,
// problem_description.cpp:1900-1939) on top of the oracle, for tests/test_avoid_singularity.py.  Built on the oracle's
// public pieces and linked against liboracle.so: the oracle builds the problem of every other term, then the objects of
// the avoid_singularity terms are appended as CostFromErrFunc (ABS) / ConstraintFromErrFunc (INEQ) objects.  That is
// their place in OptProb order as long as the avoid_singularity terms come last in the description, which the entry
// points require.
//
// err = 1/(s + lambda) - 1/(0.1 + lambda), s the smallest singular value of the 6 x D geometric Jacobian of the link's
// origin, by a one-sided Jacobi SVD (the rotation order and stopping rule of the device's); the gradient is the
// reference's forward difference g_j = u' ((J(q + eps e_j) - J(q)) / eps) v, eps = 1e-6, times -1 / (s + lambda)^2.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>

#include "trajopt.hpp"

using namespace oracle;

namespace {
thread_local std::string g_err;
constexpr double kEps = 1e-6, kUlp = 2.220446049250313e-16;  // rotations stop at |a_p.a_q| <= M kUlp |a_p||a_q|
constexpr int kSweeps = 32;

// J: [6][D] row-major.  sigma: the smallest singular value, u[6], v[D] its singular vectors (the undefined one of the
// pair is 0 when sigma is 0).
void jacobiSvdMin(const double* J, int D, double& sigma, double* u, double* v) {
  const int NC = D < 6 ? D : 6, M = D < 6 ? 6 : D;
  std::vector<double> A(static_cast<size_t>(M) * NC), V(static_cast<size_t>(NC) * NC, 0.0);  // row-major
  for (int i = 0; i < M; ++i)
    for (int k = 0; k < NC; ++k) A[i * NC + k] = D < 6 ? J[i * D + k] : J[k * D + i];
  for (int k = 0; k < NC; ++k) V[k * NC + k] = 1.0;
  auto dot = [&](int p, int q) {
    double s = 0.0;
    for (int i = 0; i < M; ++i) s += A[i * NC + p] * A[i * NC + q];
    return s;
  };
  for (int sweep = 0; sweep < kSweeps; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < NC - 1; ++p)
      for (int q = p + 1; q < NC; ++q) {
        const double al = dot(p, p), be = dot(q, q), ga = dot(p, q);
        if (!(std::fabs(ga) > M * kUlp * std::sqrt(al * be))) continue;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
        for (int i = 0; i < M; ++i) {
          const double ap = A[i * NC + p], aq = A[i * NC + q];
          A[i * NC + p] = c * ap - s * aq;
          A[i * NC + q] = s * ap + c * aq;
        }
        for (int i = 0; i < NC; ++i) {
          const double vp = V[i * NC + p], vq = V[i * NC + q];
          V[i * NC + p] = c * vp - s * vq;
          V[i * NC + q] = s * vp + c * vq;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
  int kmin = 0;
  sigma = 0.0;
  for (int k = 0; k < NC; ++k) {
    const double sk = std::sqrt(dot(k, k));
    if (k == 0 || sk < sigma) {
      sigma = sk;
      kmin = k;
    }
  }
  double* w = D < 6 ? u : v;   // W_k / sigma
  double* vk = D < 6 ? v : u;  // V_k
  for (int i = 0; i < M; ++i) w[i] = sigma > 0.0 ? A[i * NC + kmin] / sigma : 0.0;
  for (int i = 0; i < NC; ++i) vk[i] = V[i * NC + kmin];
}

void jacobianAt(const Robot& robot, const double* q, int link, std::vector<double>& J) {
  std::vector<Pose> fr;
  robot.fk(q, fr);
  std::vector<Vec> Jv;
  robot.jacobian(fr, link, fr[link].p, Jv);
  const int D = robot.n_dof;
  J.assign(6 * D, 0.0);
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < D; ++j) J[i * D + j] = Jv[i][j];
}

// err and the unscaled gradient of one waypoint
void errGrad(const Robot& robot, const double* q, int link, double lambda, double* err, double* grad, double* sigma_out) {
  const int D = robot.n_dof;
  std::vector<double> J0, Jk;
  jacobianAt(robot, q, link, J0);
  double sigma, u[6], v[16];
  jacobiSvdMin(J0.data(), D, sigma, u, v);
  if (err) *err = 1.0 / (sigma + lambda) - 1.0 / (0.1 + lambda);
  if (sigma_out) *sigma_out = sigma;
  if (!grad) return;
  std::vector<double> qk(q, q + D), dJ(6 * D);
  for (int j = 0; j < D; ++j) {
    qk[j] = q[j] + kEps;
    jacobianAt(robot, qk.data(), link, Jk);
    qk[j] = q[j];
    for (int e = 0; e < 6 * D; ++e) dJ[e] = (Jk[e] - J0[e]) / kEps;  // difference matrix, then the division
    double g = 0.0;
    for (int c = 0; c < D; ++c) {  // (u' dJ) v
      double s = 0.0;
      for (int i = 0; i < 6; ++i) s += u[i] * dJ[i * D + c];
      g += s * v[c];
    }
    grad[j] = g;
  }
  const double scale = -1.0 / ((sigma + lambda) * (sigma + lambda));
  for (int j = 0; j < D; ++j) grad[j] *= scale;
}

struct Built {
  TrajProblem tp;
  int n_cart_rows = 0, cart_stride = 0;
  std::vector<std::pair<int, int>> sing;  // (term, step) of every avoid_singularity object, in cart-row order
};

Built build(const tb200_problem_desc& d, int b) {
  std::vector<tb200_term> rest;
  std::vector<int> sing_terms;
  for (int k = 0; k < d.n_terms; ++k) {
    if (d.terms[k].kind == TB200_TERM_AVOID_SINGULARITY) {
      sing_terms.push_back(k);
    } else {
      if (!sing_terms.empty()) throw std::runtime_error("avoid_singularity terms must come last");
      rest.push_back(d.terms[k]);
    }
  }
  tb200_problem_desc d2 = d;
  d2.terms = rest.data();
  d2.n_terms = static_cast<int>(rest.size());
  Built out;
  out.tp = buildProblem(d2, b, tb200inl_cast_rows_per_pair(&d));
  const int D = d.robot.n_dof;
  bool has_vel = false;
  for (const tb200_term& t : rest) {
    if (t.kind == TB200_TERM_CART_POSE) {
      for (int i = 0; i < 3; ++i) out.n_cart_rows += std::fabs(t.pos_coeffs[i]) > 1e-5;
      for (int i = 0; i < 3; ++i) out.n_cart_rows += std::fabs(t.rot_coeffs[i]) > 1e-5;
    } else if (t.kind == TB200_TERM_CART_VEL) {
      out.n_cart_rows += 6 * (t.last_step - t.first_step + 1);
      has_vel = true;
    }
  }
  out.cart_stride = has_vel ? 2 * D : D;
  auto robot = out.tp.robot;
  for (int k : sing_terms) {
    const tb200_term& t = d.terms[k];
    if (t.link < 0 || t.link >= d.robot.n_segments) throw std::runtime_error("avoid_singularity link out of range");
    if (t.first_step < 0 || t.last_step >= d.n_steps || t.first_step > t.last_step)
      throw std::runtime_error("avoid_singularity steps outside the trajectory");
    const int link = t.link;
    const double lambda = t.lambda;
    for (int s = t.first_step; s <= t.last_step; ++s) {
      std::vector<int> vars(D);
      for (int j = 0; j < D; ++j) vars[j] = s * D + j;
      VectorFn f = [robot, link, lambda](const Vec& q) {
        Vec e(1);
        errGrad(*robot, q.data(), link, lambda, &e[0], nullptr, nullptr);
        return e;
      };
      MatrixFn dfdx = [robot, link, lambda](const Vec& q) {
        std::vector<Vec> g(1, Vec(q.size()));
        errGrad(*robot, q.data(), link, lambda, nullptr, g[0].data(), nullptr);
        return g;
      };
      const std::string name = "avoid_singularity_" + std::to_string(s);
      if (t.role == TB200_ROLE_COST) {
        auto c = std::make_shared<CostFromErrFunc>(f, dfdx, vars, Vec{t.coeffs[0]}, ABS);
        c->name = name;
        out.tp.prob->addCost(c);
        out.tp.cost_names.push_back(name);
      } else {
        auto c = std::make_shared<ConstraintFromErrFunc>(f, dfdx, vars, Vec{t.coeffs[0]}, INEQ);
        c->name = name;
        out.tp.prob->addConstraint(c);
        out.tp.cnt_names.push_back(name);
      }
      out.sing.push_back({k, s});
    }
  }
  return out;
}
}  // namespace

extern "C" {

const char* aso_last_error() { return g_err.c_str(); }

// sigma, u[6], v[D] of a 6 x D matrix (row-major)
int aso_svd_min(const double* J, int D, double* sigma, double* u, double* v) {
  jacobiSvdMin(J, D, *sigma, u, v);
  return 0;
}

// the Jacobian, sigma, err and the unscaled gradient of one waypoint
int aso_err_grad(const tb200_robot* r, const double* q, int link, double lambda, double* J, double* sigma, double* err,
                 double* grad) {
  try {
    Robot robot(*r);
    std::vector<double> Jv;
    jacobianAt(robot, q, link, Jv);
    if (J) std::memcpy(J, Jv.data(), sizeof(double) * Jv.size());
    errGrad(robot, q, link, lambda, err, grad, sigma);
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// [0] n_costs, [1] n_cnts, [2] n_cart_rows, [3] cart_stride
int aso_layout(const tb200_problem_desc* d, int32_t* out) {
  try {
    Built bl = build(*d, 0);
    out[0] = static_cast<int>(bl.tp.cost_names.size());
    out[1] = static_cast<int>(bl.tp.cnt_names.size());
    out[2] = bl.n_cart_rows + static_cast<int>(bl.sing.size());
    out[3] = bl.cart_stride;
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// the avoid_singularity objects in OptProb order: is_cnt (0 cost, 1 constraint), index in its list, term, step; returns
// their number (<= cap)
int aso_sing_objects(const tb200_problem_desc* d, int cap, int32_t* is_cnt, int32_t* index, int32_t* term, int32_t* step) {
  try {
    Built bl = build(*d, 0);
    int nc = static_cast<int>(bl.tp.cost_names.size()), nk = static_cast<int>(bl.tp.cnt_names.size()), n = 0;
    int c_at = nc, k_at = nk;
    for (auto [k, s] : bl.sing) (d->terms[k].role == TB200_ROLE_COST ? c_at : k_at) -= 1;
    for (auto [k, s] : bl.sing) {
      if (n >= cap) break;
      const bool cnt = d->terms[k].role != TB200_ROLE_COST;
      is_cnt[n] = cnt;
      index[n] = cnt ? k_at++ : c_at++;
      term[n] = k;
      step[n] = s;
      ++n;
    }
    return n;
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// cart rows (every term's, the avoid_singularity rows last), exact cost values and violations at x
int aso_convexify_batch(const tb200_problem_desc* d, int b0, int b1, const double* x, double* cart_err, double* cart_jac,
                        double* cost_vals, double* cnt_viols) {
  const int T = d->n_steps, D = d->robot.n_dof;
  try {
    for (int b = b0; b < b1; ++b) {
      Built bl = build(*d, b);
      const int R = bl.n_cart_rows + static_cast<int>(bl.sing.size()), CS = bl.cart_stride;
      Vec xv(x + static_cast<size_t>(b) * T * D, x + static_cast<size_t>(b + 1) * T * D);
      Vec err;
      std::vector<Vec> jac;
      for (auto& h : bl.tp.cart_hooks) h(xv, err, jac);
      for (auto [k, s] : bl.sing) {
        const tb200_term& t = d->terms[k];
        double e, g[16];
        errGrad(*bl.tp.robot, xv.data() + s * D, t.link, t.lambda, &e, g, nullptr);
        err.push_back(t.coeffs[0] * e);
        Vec row(D);
        for (int j = 0; j < D; ++j) row[j] = t.coeffs[0] * g[j];
        jac.push_back(row);
      }
      for (int r = 0; r < R; ++r) {
        cart_err[static_cast<size_t>(b) * R + r] = err[r];
        double* o = cart_jac + (static_cast<size_t>(b) * R + r) * CS;
        for (int j = 0; j < CS; ++j) o[j] = j < static_cast<int>(jac[r].size()) ? jac[r][j] : 0.0;
      }
      const auto& costs = bl.tp.prob->getCosts();
      for (size_t i = 0; i < costs.size(); ++i) cost_vals[b * costs.size() + i] = costs[i]->value(xv);
      const auto cnts = bl.tp.prob->getConstraints();
      for (size_t i = 0; i < cnts.size(); ++i) cnt_viols[b * cnts.size() + i] = cnts[i]->violation(xv);
    }
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// one QP convexified at x (as oracle_qp_solve_batch)
int aso_qp_solve_batch(const tb200_problem_desc* d, int b0, int b1, const double* x, const double* trust,
                       const double* merit_coeffs, double* new_x, int32_t* qp_status, double* model_cost_vals,
                       double* model_cnt_viols) {
  const int N = d->n_steps * d->robot.n_dof;
  try {
    for (int b = b0; b < b1; ++b) {
      Built bl = build(*d, b);
      Model* model = bl.tp.prob->model();
      const auto& costs = bl.tp.prob->getCosts();
      const auto cnts = bl.tp.prob->getConstraints();
      Vec xv(x + static_cast<size_t>(b) * N, x + static_cast<size_t>(b + 1) * N);
      std::vector<std::shared_ptr<ConvexObjective>> cm, ccm;
      std::vector<std::shared_ptr<ConvexConstraints>> km;
      for (auto& c : costs) cm.push_back(c->convex(xv, model));
      for (auto& c : cnts) km.push_back(c->convex(xv, model));
      for (size_t c = 0; c < km.size(); ++c) {
        auto obj = std::make_shared<ConvexObjective>(model);
        const double mu = merit_coeffs[b * cnts.size() + c];
        for (const AffExpr& a : km[c]->eqs) obj->addAbs(a, mu);
        for (const AffExpr& a : km[c]->ineqs) obj->addHinge(a, mu);
        ccm.push_back(obj);
      }
      for (auto& c : cm) c->addConstraintsToModel();
      for (auto& c : ccm) c->addConstraintsToModel();
      QuadExpr obj;
      for (auto& c : cm) exprInc(obj, c->quad);
      for (auto& c : ccm) exprInc(obj, c->quad);
      model->setObjective(obj);
      for (int i = 0; i < N; ++i) {
        const double lb = bl.tp.prob->lower()[i], ub = bl.tp.prob->upper()[i];
        const double xi = std::min(std::max(xv[i], lb), ub);
        model->setVarBounds(i, std::max(xi - trust[b], lb), std::min(xi + trust[b], ub));
      }
      const CvxStatus st = model->optimize();
      const Vec& sol = model->solution();
      std::memcpy(new_x + static_cast<size_t>(b) * N, sol.data(), sizeof(double) * N);
      qp_status[b] = st;
      for (size_t i = 0; i < cm.size(); ++i) model_cost_vals[b * cm.size() + i] = cm[i]->value(sol.data());
      for (size_t i = 0; i < km.size(); ++i) model_cnt_viols[b * km.size() + i] = km[i]->violation(sol.data());
    }
    return 0;
  } catch (const std::exception& e) {
    g_err = e.what();
    return 1;
  }
}

// BasicTrustRegionSQP::optimize() per trajectory (as oracle_solve_batch; OpenMP over trajectories)
// trace (optional): [B][trace_cap][14] the driver's decision trace per trajectory (TraceEntry columns), trace_len [B]
int aso_solve_batch(const tb200_problem_desc* d, int b0, int b1, double* x, int32_t* status, double* total_cost,
                    double* cost_vals, double* cnt_viols, int32_t* n_qp_solves, int32_t* n_func_evals, double* trace,
                    int trace_cap, int32_t* trace_len) {
  const int N = d->n_steps * d->robot.n_dof;
  int err = 0;
#pragma omp parallel for schedule(dynamic)
  for (int b = b0; b < b1; ++b) {
    try {
      Built bl = build(*d, b);
      BasicTrustRegionSQP opt(bl.tp.prob);
      opt.params() = sqpParamsFrom(d->sqp);
      opt.initialize(bl.tp.init);
      opt.optimize();
      const OptResults& r = opt.results();
      const size_t nc = bl.tp.cost_names.size(), nk = bl.tp.cnt_names.size();
      std::memcpy(x + static_cast<size_t>(b) * N, r.x.data(), sizeof(double) * N);
      status[b] = r.status;
      total_cost[b] = r.total_cost;
      for (size_t i = 0; i < nc; ++i) cost_vals[b * nc + i] = r.cost_vals[i];
      for (size_t i = 0; i < nk; ++i) cnt_viols[b * nk + i] = r.cnt_viols[i];
      n_qp_solves[b] = r.n_qp_solves;
      n_func_evals[b] = r.n_func_evals;
      if (trace) {
        int n = 0;
        for (const TraceEntry& te : opt.trace) {
          if (n >= trace_cap) break;
          double* o = trace + (static_cast<size_t>(b) * trace_cap + n) * 14;
          o[0] = te.merit_round; o[1] = te.iter; o[2] = te.trust; o[3] = te.old_merit; o[4] = te.model_merit;
          o[5] = te.new_merit; o[6] = te.qp_status; o[7] = te.admm_iters; o[8] = te.action;
          o[9] = te.pri; o[10] = te.dua; o[11] = te.rho; o[12] = te.polish; o[13] = te.warm;
          ++n;
        }
        trace_len[b] = n;
      }
    } catch (const std::exception& e) {
#pragma omp critical
      {
        g_err = e.what();
        err = 1;
      }
    }
  }
  return err;
}
}
