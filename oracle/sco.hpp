// ORACLE — TEST INFRASTRUCTURE ONLY.  Nothing under trajopt_b200/ (the product) may include,
// link or call this.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference leg use it, as the checker / the timed CPU baseline.
//
// CPU fp64 restatement of the reference's sequential-convex-optimisation core
// (tesseract-robotics/trajopt, trajopt_sco/), written from scratch:
//   * expression algebra          trajopt_sco/src/expr_ops.cpp:55-99, solver_interface.cpp:92-109
//   * penalty reformulation       trajopt_sco/src/modeling.cpp:18-51, 86-97, 132-169
//   * QP canonical form           trajopt_sco/src/osqp_interface.cpp:170-281, solver_utils.cpp:49-144
//   * trust-region SQP driver     trajopt_sco/src/optimizers.cpp:59-81, 151-170, 380-426, 699-991
//   * err-func wrapping / numdiff trajopt_sco/src/modeling_utils.cpp:31-269, num_diff.cpp:40-105
// The QP arithmetic itself lives in OSQP v1.0.0 (pinned by trajopt_ext/osqp/CMakeLists.txt:7,32),
// which is NOT in the reference tree; qp_solve() restates its published ADMM algorithm
// (Stellato et al., "OSQP: an operator splitting solver for quadratic programs", 2020) with the
// reference's settings (osqp_interface.cpp:78-90).  PARITY STATUS: the SQP driver, the QP
// canonical form and the expression algebra are pinned by the reference's own known-answer tests
// (tests/test_oracle_golden.py); the ADMM iterates are "parity unpinned" against real OSQP (no
// OSQP binary, and OSQP's default adaptive-rho schedule is wall-clock dependent) — they are
// pinned only through QP optimality (KKT residual checks) and the behavioural end-state tests.
#pragma once
#include <cmath>
#include <cstdint>
#include <functional>
#include <limits>
#include <memory>
#include <string>
#include <vector>

namespace oracle {

using Vec = std::vector<double>;
constexpr double kInf = std::numeric_limits<double>::infinity();

// ---------------------------------------------------------------- expressions
// sco::AffExpr / sco::QuadExpr (solver_interface.hpp:181-219) with variables as plain indices.
struct AffExpr {
  double constant = 0.0;
  std::vector<int> vars;
  Vec coeffs;
  AffExpr() = default;
  explicit AffExpr(double c) : constant(c) {}
  static AffExpr var(int v) {
    AffExpr a;
    a.vars.push_back(v);
    a.coeffs.push_back(1.0);
    return a;
  }
  double value(const double* x) const;
};
struct QuadExpr {
  AffExpr aff;
  std::vector<int> v1, v2;
  Vec coeffs;
  double value(const double* x) const;  // aff + sum c_k x[v1_k] x[v2_k]
};
AffExpr cleanupAff(const AffExpr& a);                 // expr_ops.cpp:86-99 (drops |c| <= 1e-7)
QuadExpr exprSquare(const AffExpr& a);                // expr_ops.cpp:55-84
void exprScale(AffExpr& a, double s);
void exprScale(QuadExpr& q, double s);
void exprInc(AffExpr& a, const AffExpr& b);
void exprInc(QuadExpr& a, const QuadExpr& b);
void exprInc(QuadExpr& a, const AffExpr& b);

// ---------------------------------------------------------------- sparse helpers
struct Csr {  // row-compressed
  int rows = 0, cols = 0;
  std::vector<int> ptr{0}, idx;
  Vec val;
  void addRow(const std::vector<int>& c, const Vec& v);
  int nnz() const { return static_cast<int>(idx.size()); }
};

// QP in OSQP canonical form: min 1/2 x'Px + q'x  s.t. l <= Ax <= u.  P given by its upper
// triangle (row i holds columns j >= i), as osqp_interface.cpp:178-180 passes it.
struct QP {
  int n = 0, m = 0;
  Csr Pu;
  Vec q;
  Csr A;
  Vec l, u;
};

// exprToEigen restated (solver_utils.cpp:12-144): dense outputs for the unit tests.
void affToRow(const AffExpr& e, int n_vars, Vec& dense_row);
void quadToDense(const QuadExpr& e, int n_vars, bool matrix_is_halved, bool force_diagonal, Vec& dense_Q,
                 Vec& q, int& nnz);
// eigenToCSC restated (solver_utils.hpp:104-153): column-compressed arrays of a dense matrix
// (explicit zeros skipped), optionally upper triangle only.
void denseToCsc(const Vec& M, int rows, int cols, bool upper_only, std::vector<long long>& row_idx,
                std::vector<long long>& col_ptr, Vec& data);

// ---------------------------------------------------------------- QP solver (OSQP-equivalent)
struct QPSettings {
  double rho = 0.1, sigma = 1e-6, alpha = 1.6;
  double eps_abs = 1e-4, eps_rel = 1e-6;          // osqp_interface.cpp:83-84
  double eps_prim_inf = 1e-4, eps_dual_inf = 1e-4;
  double delta = 1e-6, adaptive_rho_tolerance = 5.0;
  int max_iter = 8192;                             // osqp_interface.cpp:85
  int scaling = 10, check_termination = 25;
  int adaptive_rho = 1, adaptive_rho_interval = 50;
  int polishing = 1, polish_refine_iter = 3;       // osqp_interface.cpp:86
  int warm_starting = 1;
  int verify_rounds = 3;     // verified-polish retries with 10x tighter ADMM tolerances (0 = plain OSQP polish)
  double verify_tol = 1e-9;  // KKT verification: primal feasibility and multiplier-sign tolerance
  int early_polish_every = 0;  // >0: also try the (verified) polish every this many iterations (optimisation O1)
  int early_polish_from = 50;
  int early_polish_stable = 1; // only try when the active-set guess is unchanged since the previous test and has not failed yet
  int warm_polished_duals = 0; // 1: warm start the next QP from the POLISHED duals as OSQP / the reference do (deviation D1 off)
};
enum QPStatus {
  QP_SOLVED = 1,
  QP_SOLVED_INACCURATE = 2,
  QP_PRIMAL_INFEASIBLE = 3,
  QP_PRIMAL_INFEASIBLE_INACCURATE = 4,
  QP_DUAL_INFEASIBLE = 5,
  QP_DUAL_INFEASIBLE_INACCURATE = 6,
  QP_MAX_ITER_REACHED = 7,
  QP_NON_CVX = 8,
  QP_UNSOLVED = 0
};
struct QPWarmStart {
  bool valid = false;
  Vec x, y;
  double rho = 0.1;
};
struct QPResult {
  int status = QP_UNSOLVED;
  Vec x, y;
  Vec y_admm;  // duals of the last ADMM iterate (before polish): what the next solve is warm-started from
  int iters = 0;
  int rho_updates = 0;
  int polish = 0;  // 1 accepted (KKT fixed point), 2 accepted by residual rule only, -1 rejected, 0 not attempted
  int pdas = 0;    // verified-polish rounds used
  int early_tries = 0;
  double pri_res = 0, dua_res = 0;
  double admm_pri = 0, admm_dua = 0;
  double rho = 0.1;
  int warm = 0;
};
QPResult qp_solve(const QP& qp, const QPSettings& s, const QPWarmStart* warm);
// KKT residuals of (x,y) for `qp` in the original (unscaled) space; used by the tests.
void qp_kkt_residuals(const QP& qp, const Vec& x, const Vec& y, double& stationarity, double& primal,
                      double& complementarity);

// ---------------------------------------------------------------- model (sco::Model + OSQPModel)
enum CvxStatus { CVX_SOLVED = 0, CVX_INFEASIBLE = 1, CVX_FAILED = 2 };
enum CntType { EQ = 0, INEQ = 1 };

class Model {
public:
  explicit Model(const QPSettings& s = QPSettings()) : settings_(s) {}
  int addVar(double lb = -kInf, double ub = kInf);
  void addEqCnt(const AffExpr& e) { addCnt(e, EQ); }     // e == 0
  void addIneqCnt(const AffExpr& e) { addCnt(e, INEQ); } // e <= 0
  // The reference removes the previous iteration's aux vars / rows lazily and compacts in update()
  // (osqp_interface.cpp:372-418); the net effect is a truncation back to the permanent content.
  void markPermanent() { n_perm_vars_ = numVars(); n_perm_cnts_ = numCnts(); }
  void truncateToPermanent();
  void setVarBounds(int var, double lb, double ub) { lbs_[var] = lb; ubs_[var] = ub; }
  void setObjective(const QuadExpr& q) { objective_ = q; }
  int numVars() const { return static_cast<int>(lbs_.size()); }
  int numCnts() const { return static_cast<int>(cnt_exprs_.size()); }
  CvxStatus optimize();
  const Vec& solution() const { return solution_; }
  void buildQP(QP& qp) const;  // osqp_interface.cpp:170-281
  const QPResult& lastResult() const { return last_; }
  QPSettings& settings() { return settings_; }
  long totalAdmmIters() const { return total_iters_; }

private:
  void addCnt(const AffExpr& e, CntType t) {
    cnt_exprs_.push_back(e);
    cnt_types_.push_back(t);
  }
  QPSettings settings_;
  Vec lbs_, ubs_;
  std::vector<AffExpr> cnt_exprs_;
  std::vector<CntType> cnt_types_;
  QuadExpr objective_;
  Vec solution_;
  int n_perm_vars_ = 0, n_perm_cnts_ = 0;
  // createOrUpdateSolver() bookkeeping (osqp_interface.cpp:283-370)
  QPResult last_;
  bool have_last_ = false;
  int last_n_ = -1, last_m_ = -1, last_nnzP_ = -1, last_nnzA_ = -1;
  long total_iters_ = 0;
};

// ---------------------------------------------------------------- convex pieces (modeling.hpp)
struct ConvexObjective {  // modeling.cpp:15-110
  explicit ConvexObjective(Model* m) : model(m) {}
  Model* model;
  QuadExpr quad;
  std::vector<AffExpr> eqs, ineqs;
  void addAffExpr(const AffExpr& a) { exprInc(quad, a); }
  void addQuadExpr(const QuadExpr& q) { exprInc(quad, q); }
  void addHinge(const AffExpr& a, double coeff);
  void addAbs(const AffExpr& a, double coeff);
  void addConstraintsToModel();
  double value(const double* x) const { return quad.value(x); }
};
struct ConvexConstraints {  // modeling.cpp:112-147
  std::vector<AffExpr> eqs, ineqs;
  Vec violations(const double* x) const;
  double violation(const double* x) const;
};

class Cost {
public:
  virtual ~Cost() = default;
  virtual double value(const Vec& x) = 0;
  virtual std::shared_ptr<ConvexObjective> convex(const Vec& x, Model* model) = 0;
  std::string name;
  int term = -1, step = -1;  // the description term and step the object was made for
};
class Constraint {
public:
  virtual ~Constraint() = default;
  virtual CntType type() const = 0;
  virtual Vec value(const Vec& x) = 0;
  virtual std::shared_ptr<ConvexConstraints> convex(const Vec& x, Model* model) = 0;
  Vec violations(const Vec& x);       // modeling.cpp:150-167
  double violation(const Vec& x);     // modeling.cpp:169
  std::string name;
  int term = -1, step = -1;  // the description term and step the object was made for
};

class OptProb {  // modeling.cpp:170-271
public:
  explicit OptProb(const QPSettings& s = QPSettings()) : model_(std::make_shared<Model>(s)) {}
  std::vector<int> createVariables(int count, const Vec& lb, const Vec& ub);
  std::vector<int> createVariables(int count);
  void addCost(std::shared_ptr<Cost> c) { costs_.push_back(std::move(c)); }
  void addConstraint(std::shared_ptr<Constraint> c);
  void addLinearConstraint(const AffExpr& e, CntType t);  // permanent model row, modeling.cpp:243-249
  std::vector<std::shared_ptr<Constraint>> getConstraints() const;  // EQ first, then INEQ
  const std::vector<std::shared_ptr<Cost>>& getCosts() const { return costs_; }
  Vec getClosestFeasiblePoint(const Vec& x, double delta = 1e-3) const;  // quirk kept: modeling.cpp:267-268
  int numVars() const { return static_cast<int>(lb_.size()); }
  const Vec& lower() const { return lb_; }
  const Vec& upper() const { return ub_; }
  Model* model() { return model_.get(); }

private:
  std::shared_ptr<Model> model_;
  Vec lb_, ub_;
  std::vector<std::shared_ptr<Cost>> costs_;
  std::vector<std::shared_ptr<Constraint>> eqcnts_, ineqcnts_;
};

// ---------------------------------------------------------------- func wrapping (modeling_utils.cpp)
using ScalarFn = std::function<double(const Vec&)>;
using VectorFn = std::function<Vec(const Vec&)>;
using MatrixFn = std::function<std::vector<Vec>(const Vec&)>;  // rows
enum PenaltyType { SQUARED, ABS, HINGE };

std::vector<Vec> calcForwardNumJac(const VectorFn& f, const Vec& x, double eps);  // num_diff.cpp:55-68

class CostFromFunc : public Cost {  // modeling_utils.cpp:41-113
public:
  CostFromFunc(ScalarFn f, std::vector<int> vars, bool full_hessian = false)
    : f_(std::move(f)), vars_(std::move(vars)), full_hessian_(full_hessian) {}
  double value(const Vec& x) override;
  std::shared_ptr<ConvexObjective> convex(const Vec& x, Model* model) override;

private:
  ScalarFn f_;
  std::vector<int> vars_;
  bool full_hessian_;
  double epsilon_ = 1e-5;
};
class CostFromErrFunc : public Cost {  // modeling_utils.cpp:115-211
public:
  CostFromErrFunc(VectorFn f, MatrixFn dfdx, std::vector<int> vars, Vec coeffs, PenaltyType pen)
    : f_(std::move(f)), dfdx_(std::move(dfdx)), vars_(std::move(vars)), coeffs_(std::move(coeffs)), pen_(pen) {}
  double value(const Vec& x) override;
  std::shared_ptr<ConvexObjective> convex(const Vec& x, Model* model) override;

private:
  VectorFn f_;
  MatrixFn dfdx_;
  std::vector<int> vars_;
  Vec coeffs_;
  PenaltyType pen_;
  double epsilon_ = 1e-5;
};
class ConstraintFromErrFunc : public Constraint {  // modeling_utils.cpp:213-269
public:
  ConstraintFromErrFunc(VectorFn f, MatrixFn dfdx, std::vector<int> vars, Vec coeffs, CntType t)
    : f_(std::move(f)), dfdx_(std::move(dfdx)), vars_(std::move(vars)), coeffs_(std::move(coeffs)), type_(t) {}
  CntType type() const override { return type_; }
  Vec value(const Vec& x) override;
  std::shared_ptr<ConvexConstraints> convex(const Vec& x, Model* model) override;

private:
  VectorFn f_;
  MatrixFn dfdx_;
  std::vector<int> vars_;
  Vec coeffs_;
  CntType type_;
  double epsilon_ = 1e-5;
};

// ---------------------------------------------------------------- SQP driver (optimizers.cpp)
enum OptStatus { OPT_CONVERGED = 0, OPT_SCO_ITERATION_LIMIT, OPT_PENALTY_ITERATION_LIMIT, OPT_TIME_LIMIT, OPT_FAILED, OPT_INVALID };

struct SQPParams {  // optimizers.hpp:92-135
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
};
struct OptResults {  // optimizers.hpp:40-59
  Vec x;
  OptStatus status = OPT_INVALID;
  double total_cost = 0;
  Vec cost_vals, cnt_viols;
  int n_func_evals = 0, n_qp_solves = 0;
};
// One accept/reject decision of the trust-region loop, for decision-trace parity tests.
struct TraceEntry {
  int merit_round, iter;
  double trust, old_merit, model_merit, new_merit;
  int qp_status, admm_iters, action;  // action: 0 shrink, 1 accept, 2 converged(small improve), 3 qp failure
  double pri = 0, dua = 0, rho = 0;
  int polish = 0, warm = 0;
};

// One entry of the iteration log.  Record 0 is the state after the first evaluation (the clamped start, its exact
// values, the initial merit coefficients); record k >= 1 is the QP solve of trace[k - 1]: the merit coefficients in
// force, the model value of every object at the QP solution, the exact values there and the point.  What a record
// does not have (record 0's model values; a failed QP's model values, exact values and point) is NaN.
struct IterRecord {
  Vec merit_coeffs, model_cost_vals, model_cnt_viols, cost_vals, cnt_viols, x;
};

void trustBox(double x, double lb, double ub, double trust, double& lo, double& hi);  // optimizers.cpp:163-168
// every variable's trust box around x (setTrustBoxConstraints, optimizers.cpp:151-170)
void setTrustBoxConstraints(OptProb& prob, const Vec& x, double trust);

// The QP of one SQP iteration at x (optimizers.cpp:781-799): the previous iteration's aux vars / rows dropped, every
// cost and constraint convexified, the constraints made costs with their merit coefficients (cntsToCosts,
// optimizers.cpp:59-81), their rows added to the model and the summed objective set.  The trust box is not set.
struct ConvexModels {
  std::vector<std::shared_ptr<ConvexObjective>> costs;
  std::vector<std::shared_ptr<ConvexConstraints>> cnts;
  // the model's values at x: the costs' values and the constraints' violations
  void values(const double* x, Vec& cost_vals, Vec& cnt_viols) const;
};
ConvexModels convexifyProblem(OptProb& prob, const Vec& x, const double* merit_coeffs);

class BasicTrustRegionSQP {
public:
  // When the run stops early (optimizers.cpp:738-753): never, on a steady_clock started in optimize() past max_time,
  // or at the first iteration top with n_qp_solves >= qp_budget.
  enum StopRule { STOP_NONE, STOP_WALL_CLOCK, STOP_QP_BUDGET };

  explicit BasicTrustRegionSQP(std::shared_ptr<OptProb> prob) : prob_(std::move(prob)) {}
  SQPParams& params() { return param_; }
  void initialize(const Vec& x) { results_ = OptResults(); results_.x = x; }
  void setStopRule(StopRule rule, double max_time, int qp_budget) {
    stop_ = rule;
    max_time_ = max_time;
    qp_budget_ = qp_budget;
  }
  OptStatus optimize();  // optimizers.cpp:699-991
  const OptResults& results() const { return results_; }
  std::vector<TraceEntry> trace;
  bool ended = false;                // the stop rule ended the run
  bool record = false;               // fill `records`
  std::vector<IterRecord> records;

private:
  std::shared_ptr<OptProb> prob_;
  SQPParams param_;
  OptResults results_;
  StopRule stop_ = STOP_NONE;
  double max_time_ = 0;
  int qp_budget_ = 0;
};

}  // namespace oracle
