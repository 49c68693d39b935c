// trajopt_b200_sco.hpp — the convex-solver plugin surface of trajopt_sco, header only, over the C ABI.
//
// Mirrors trajopt_sco/include/trajopt_sco/solver_interface.hpp:40-290 by name: sco::Var / Cnt / AffExpr / QuadExpr,
// sco::Model with addVar / addEqCnt / addIneqCnt / removeVars / removeCnts / update / setVarBounds / setObjective /
// optimize / getVarValues / writeToFile / getVars, sco::ModelType, sco::createModel(ModelType).  A caller of the
// reference's sco layer (its BasicTrustRegionSQP, or any code that builds QPs through sco::Model) gets the GPU QP
// solver as its back end by including this header and linking libtrajopt_b200.so: createModel() returns a model whose
// optimize() assembles OSQP's canonical form exactly as OSQPModel does (osqp_interface.cpp:170-281: P = M + M', upper
// triangle; A = [constraint rows; I]; EQ rows before nothing in particular — row order is insertion order) and hands it to
// tb200_qp_solve_general (include/trajopt_b200.h).  Status map as osqp_interface.cpp:565-614.
//
// Differences, on purpose: ModelType names are resolved BY NAME (the reference's name table is permuted against its enum,
// solver_interface.cpp:14 vs solver_interface.hpp:229-236, so ModelType("OSQP") there yields QPOASES); every solver name
// maps to the one back end this library has.  A quadratic inequality throws "NOT IMPLEMENTED" like OSQPModel
// (osqp_interface.cpp:150).
#pragma once
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <fstream>
#include <memory>
#include <mutex>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "trajopt_b200.h"

namespace sco {

using DblVec = std::vector<double>;
using IntVec = std::vector<int>;
using SizeTVec = std::vector<std::size_t>;

enum ConstraintType : std::uint8_t { EQ, INEQ };
enum CvxOptStatus : std::uint8_t { CVX_SOLVED, CVX_INFEASIBLE, CVX_FAILED };

struct VarRep {
  using Ptr = std::shared_ptr<VarRep>;
  VarRep(std::size_t _index, std::string _name, void* _creator) : index(_index), name(std::move(_name)), creator(_creator) {}
  std::size_t index;
  std::string name;
  bool removed{ false };
  void* creator;
};
struct Var {
  VarRep::Ptr var_rep{ nullptr };
  Var() = default;
  Var(VarRep::Ptr rep) : var_rep(std::move(rep)) {}  // NOLINT
  double value(const double* x) const { return x[var_rep->index]; }
  double value(const DblVec& x) const {
    assert(var_rep->index < x.size());
    return x[var_rep->index];
  }
};
struct CntRep {
  using Ptr = std::shared_ptr<CntRep>;
  CntRep(std::size_t _index, void* _creator) : index(_index), creator(_creator) {}
  std::size_t index;
  bool removed{ false };
  void* creator;
  ConstraintType type{ ConstraintType::EQ };
  std::string expr;
};
struct Cnt {
  CntRep::Ptr cnt_rep{ nullptr };
  Cnt() = default;
  Cnt(CntRep::Ptr rep) : cnt_rep(std::move(rep)) {}  // NOLINT
};
using VarVector = std::vector<Var>;
using CntVector = std::vector<Cnt>;

struct AffExpr {
  double constant{ 0 };
  DblVec coeffs;
  VarVector vars;
  AffExpr() = default;
  explicit AffExpr(double a) : constant(a) {}
  explicit AffExpr(const Var& v) : coeffs(1, 1.0), vars(1, v) {}
  std::size_t size() const { return coeffs.size(); }
  double value(const double* x) const {
    double out = constant;
    for (std::size_t i = 0; i < size(); ++i) out += coeffs[i] * vars[i].value(x);
    return out;
  }
  double value(const DblVec& x) const { return value(x.data()); }
};
struct QuadExpr {
  AffExpr affexpr;
  DblVec coeffs;
  VarVector vars1;
  VarVector vars2;
  QuadExpr() = default;
  explicit QuadExpr(double a) : affexpr(a) {}
  explicit QuadExpr(const Var& v) : affexpr(v) {}
  explicit QuadExpr(AffExpr aff) : affexpr(std::move(aff)) {}
  std::size_t size() const { return coeffs.size(); }
  double value(const double* x) const {
    double out = affexpr.value(x);
    for (std::size_t i = 0; i < size(); ++i) out += coeffs[i] * vars1[i].value(x) * vars2[i].value(x);
    return out;
  }
  double value(const DblVec& x) const { return value(x.data()); }
};

inline std::ostream& operator<<(std::ostream& o, const Var& v) { return o << (v.var_rep ? v.var_rep->name : std::string("nullvar")); }
inline std::ostream& operator<<(std::ostream& o, const Cnt& c) { return o << c.cnt_rep->expr << ((c.cnt_rep->type == EQ) ? " == 0" : " <= 0"); }
inline std::ostream& operator<<(std::ostream& o, const AffExpr& e) {
  o << e.constant;
  for (std::size_t i = 0; i < e.size(); ++i) o << " + " << e.coeffs[i] << "*" << e.vars[i];
  return o;
}
inline std::ostream& operator<<(std::ostream& o, const QuadExpr& e) {
  o << e.affexpr;
  for (std::size_t i = 0; i < e.size(); ++i) o << " + " << e.coeffs[i] << "*" << e.vars1[i] << "*" << e.vars2[i];
  return o;
}

// ---- the few expression operations callers of the model use (trajopt_sco/src/expr_ops.cpp:8-99) ----------------------
inline void exprScale(AffExpr& v, double a) {
  v.constant *= a;
  for (double& c : v.coeffs) c *= a;
}
inline void exprInc(AffExpr& a, double b) { a.constant += b; }
inline void exprInc(AffExpr& a, const Var& b) {
  a.vars.push_back(b);
  a.coeffs.push_back(1.0);
}
inline void exprInc(AffExpr& a, const AffExpr& b) {
  a.constant += b.constant;
  a.coeffs.insert(a.coeffs.end(), b.coeffs.begin(), b.coeffs.end());
  a.vars.insert(a.vars.end(), b.vars.begin(), b.vars.end());
}
inline QuadExpr exprMult(const AffExpr& a, const AffExpr& b) {  // (a.c + a.k . x)(b.c + b.k . x)
  QuadExpr out;
  out.affexpr.constant = a.constant * b.constant;
  for (std::size_t i = 0; i < a.size(); ++i) {
    out.affexpr.vars.push_back(a.vars[i]);
    out.affexpr.coeffs.push_back(b.constant * a.coeffs[i]);
  }
  for (std::size_t i = 0; i < b.size(); ++i) {
    out.affexpr.vars.push_back(b.vars[i]);
    out.affexpr.coeffs.push_back(a.constant * b.coeffs[i]);
  }
  for (std::size_t i = 0; i < a.size(); ++i)
    for (std::size_t j = 0; j < b.size(); ++j) {
      out.vars1.push_back(a.vars[i]);
      out.vars2.push_back(b.vars[j]);
      out.coeffs.push_back(a.coeffs[i] * b.coeffs[j]);
    }
  return out;
}
inline QuadExpr exprSquare(const AffExpr& a) {  // expr_ops.cpp:55-84: diagonal terms c_i^2, off-diagonal 2 c_i c_j (i < j)
  QuadExpr out;
  out.affexpr.constant = a.constant * a.constant;
  for (std::size_t i = 0; i < a.size(); ++i) {
    out.affexpr.vars.push_back(a.vars[i]);
    out.affexpr.coeffs.push_back(2.0 * a.constant * a.coeffs[i]);
  }
  for (std::size_t i = 0; i < a.size(); ++i) {
    out.vars1.push_back(a.vars[i]);
    out.vars2.push_back(a.vars[i]);
    out.coeffs.push_back(a.coeffs[i] * a.coeffs[i]);
    for (std::size_t j = i + 1; j < a.size(); ++j) {
      out.vars1.push_back(a.vars[i]);
      out.vars2.push_back(a.vars[j]);
      out.coeffs.push_back(2.0 * a.coeffs[i] * a.coeffs[j]);
    }
  }
  return out;
}

inline void vars2inds(const VarVector& vars, SizeTVec& inds) {
  inds.resize(vars.size());
  for (std::size_t i = 0; i < inds.size(); ++i) inds[i] = vars[i].var_rep->index;
}
inline void cnts2inds(const CntVector& cnts, SizeTVec& inds) {
  inds.resize(cnts.size());
  for (std::size_t i = 0; i < inds.size(); ++i) inds[i] = cnts[i].cnt_rep->index;
}

// ---- sco::Model (solver_interface.hpp:54-104) ---------------------------------------------------------------------------
class Model {
public:
  using Ptr = std::shared_ptr<Model>;
  using ConstPtr = std::shared_ptr<const Model>;
  Model() = default;
  virtual ~Model() = default;
  virtual Var addVar(const std::string& name) = 0;
  virtual Var addVar(const std::string& name, double lb, double ub) {
    Var v = addVar(name);
    setVarBounds(v, lb, ub);
    return v;
  }
  virtual Cnt addEqCnt(const AffExpr&, const std::string& name) = 0;     // expr == 0
  virtual Cnt addIneqCnt(const AffExpr&, const std::string& name) = 0;   // expr <= 0
  virtual Cnt addIneqCnt(const QuadExpr&, const std::string& name) = 0;  // expr <= 0
  virtual void removeVar(const Var& var) { removeVars(VarVector(1, var)); }
  virtual void removeCnt(const Cnt& cnt) { removeCnts(CntVector(1, cnt)); }
  virtual void removeVars(const VarVector& vars) = 0;
  virtual void removeCnts(const CntVector& cnts) = 0;
  virtual void update() = 0;
  virtual void setVarBounds(const Var& var, double lower, double upper) { setVarBounds(VarVector(1, var), DblVec(1, lower), DblVec(1, upper)); }
  virtual void setVarBounds(const VarVector& vars, const DblVec& lower, const DblVec& upper) = 0;
  virtual double getVarValue(const Var& var) const { return getVarValues(VarVector(1, var))[0]; }
  virtual DblVec getVarValues(const VarVector& vars) const = 0;
  virtual CvxOptStatus optimize() = 0;
  virtual void setObjective(const AffExpr&) = 0;
  virtual void setObjective(const QuadExpr&) = 0;
  virtual void writeToFile(const std::string& fname) const = 0;
  virtual VarVector getVars() const = 0;
};

struct ModelConfig {
  using Ptr = std::shared_ptr<ModelConfig>;
  using ConstPtr = std::shared_ptr<const ModelConfig>;
  virtual ~ModelConfig() = default;
};
// settings of the GPU QP back end (the OSQPModelConfig of this library: osqp_interface.hpp:17-36)
struct B200ModelConfig : ModelConfig {
  tb200_qp_settings settings;
  int device = 0;
  B200ModelConfig() { tb200_default_qp_settings(&settings); }
};

class ModelType {
public:
  enum Value : std::uint8_t { GUROBI, OSQP, QPOASES, BPMPD, AUTO_SOLVER };
  ModelType() = default;
  ModelType(const ModelType::Value& v) : value_(v) {}  // NOLINT
  ModelType(const int& v) : value_(static_cast<Value>(v)) {}  // NOLINT
  ModelType(const std::string& s) {  // NOLINT  (by NAME: see the header comment)
    static const char* names[] = { "GUROBI", "OSQP", "QPOASES", "BPMPD", "AUTO_SOLVER" };
    for (int i = 0; i < 5; ++i)
      if (s == names[i]) {
        value_ = static_cast<Value>(i);
        return;
      }
    throw std::runtime_error("invalid solver name:\"" + s + "\"");
  }
  operator int() const { return static_cast<int>(value_); }  // NOLINT
  bool operator==(const ModelType::Value& a) const { return value_ == a; }
  bool operator==(const ModelType& a) const { return value_ == a.value_; }
  bool operator!=(const ModelType& a) const { return value_ != a.value_; }
  friend std::ostream& operator<<(std::ostream& os, const ModelType& cs) {
    static const char* names[] = { "GUROBI", "OSQP", "QPOASES", "BPMPD", "AUTO_SOLVER" };
    return os << names[static_cast<int>(cs.value_)];
  }

private:
  Value value_{ Value::AUTO_SOLVER };
};
inline std::vector<ModelType> availableSolvers() { return { ModelType(ModelType::OSQP) }; }

// ---- the model of this library: OSQPModel's bookkeeping (osqp_interface.cpp:123-168, 372-440, 616-643) over the GPU QP
class B200Model : public Model {
public:
  explicit B200Model(const ModelConfig::ConstPtr& config = nullptr) {
    if (auto c = std::dynamic_pointer_cast<const B200ModelConfig>(config)) config_ = *c;
  }
  Var addVar(const std::string& name) override {
    const std::scoped_lock lock(mutex_);
    vars_.emplace_back(std::make_shared<VarRep>(vars_.size(), name, this));
    lbs_.push_back(-1e30);
    ubs_.push_back(1e30);
    return vars_.back();
  }
  using Model::addVar;
  Cnt addEqCnt(const AffExpr& expr, const std::string& /*name*/) override { return addCnt(expr, EQ); }
  Cnt addIneqCnt(const AffExpr& expr, const std::string& /*name*/) override { return addCnt(expr, INEQ); }
  Cnt addIneqCnt(const QuadExpr&, const std::string& /*name*/) override { throw std::runtime_error("NOT IMPLEMENTED"); }
  void removeVars(const VarVector& vars) override {
    const std::scoped_lock lock(mutex_);
    for (const auto& var : vars) var.var_rep->removed = true;
  }
  void removeCnts(const CntVector& cnts) override {
    const std::scoped_lock lock(mutex_);
    for (const auto& cnt : cnts) cnt.cnt_rep->removed = true;
  }
  void update() override {  // osqp_interface.cpp:372-418: compact what was removed, renumber
    {
      std::size_t inew = 0;
      for (std::size_t iold = 0; iold < vars_.size(); ++iold) {
        Var& var = vars_[iold];
        if (!var.var_rep->removed) {
          vars_[inew] = var;
          lbs_[inew] = lbs_[iold];
          ubs_[inew] = ubs_[iold];
          var.var_rep->index = inew;
          ++inew;
        } else {
          var.var_rep = nullptr;
        }
      }
      vars_.resize(inew);
      lbs_.resize(inew);
      ubs_.resize(inew);
    }
    {
      std::size_t inew = 0;
      for (std::size_t iold = 0; iold < cnts_.size(); ++iold) {
        Cnt& cnt = cnts_[iold];
        if (!cnt.cnt_rep->removed) {
          cnts_[inew] = cnt;
          cnt_exprs_[inew] = cnt_exprs_[iold];
          cnt_types_[inew] = cnt_types_[iold];
          cnt.cnt_rep->index = inew;
          ++inew;
        } else {
          cnt.cnt_rep = nullptr;
        }
      }
      cnts_.resize(inew);
      cnt_exprs_.resize(inew);
      cnt_types_.resize(inew);
    }
  }
  using Model::setVarBounds;
  void setVarBounds(const VarVector& vars, const DblVec& lower, const DblVec& upper) override {
    for (std::size_t i = 0; i < vars.size(); ++i) {
      const std::size_t varind = vars[i].var_rep->index;
      lbs_[varind] = lower[i];
      ubs_[varind] = upper[i];
    }
  }
  DblVec getVarValues(const VarVector& vars) const override {
    DblVec out(vars.size());
    for (std::size_t i = 0; i < vars.size(); ++i) out[i] = solution_[vars[i].var_rep->index];
    return out;
  }
  void setObjective(const AffExpr& expr) override { objective_.affexpr = expr; }
  void setObjective(const QuadExpr& expr) override { objective_ = expr; }
  VarVector getVars() const override { return vars_; }
  void writeToFile(const std::string& fname) const override {  // osqp_interface.cpp:623-643
    std::ofstream out(fname);
    out << "\\ Generated by trajopt_sco with backend trajopt_b200\n";
    out << "Minimize\n" << objective_ << "Subject To\n";
    for (std::size_t i = 0; i < cnt_exprs_.size(); ++i) out << cnt_exprs_[i] << ((cnt_types_[i] == INEQ) ? " <= " : " = ") << 0 << "\n";
    out << "Bounds\n";
    for (std::size_t i = 0; i < vars_.size(); ++i) out << lbs_[i] << " <= " << vars_[i] << " <= " << ubs_[i] << "\n";
    out << "End";
  }

  // The QP in OSQP's canonical form as OSQPModel::updateObjective / updateConstraints build it (osqp_interface.cpp:170-281,
  // exprToEigen solver_utils.cpp:12-144): P = M + M' with M(i,j) the quadratic coefficients (full symmetric matrix here, the
  // solver reads the upper triangle), q the linear part, A = [constraint rows; I], l / u from the row types and the bounds.
  void canonicalForm(std::size_t& n, std::size_t& m, DblVec& P, DblVec& q, DblVec& A, DblVec& l, DblVec& u) const {
    n = vars_.size();
    const std::size_t mc = cnts_.size();
    m = mc + n;
    P.assign(n * n, 0.0);
    q.assign(n, 0.0);
    A.assign(m * n, 0.0);
    l.assign(m, -1e30);
    u.assign(m, 1e30);
    for (std::size_t k = 0; k < objective_.size(); ++k) {
      const std::size_t i = objective_.vars1[k].var_rep->index, j = objective_.vars2[k].var_rep->index;
      P[i * n + j] += objective_.coeffs[k];
      P[j * n + i] += objective_.coeffs[k];  // M + M': a diagonal term ends up doubled, as in exprToEigen(..., true)
    }
    for (std::size_t k = 0; k < objective_.affexpr.size(); ++k) q[objective_.affexpr.vars[k].var_rep->index] += objective_.affexpr.coeffs[k];
    for (std::size_t r = 0; r < mc; ++r) {
      const AffExpr& e = cnt_exprs_[r];
      for (std::size_t k = 0; k < e.size(); ++k) A[r * n + e.vars[k].var_rep->index] += e.coeffs[k];
      l[r] = (cnt_types_[r] == INEQ) ? -1e30 : -e.constant;
      u[r] = -e.constant;
    }
    for (std::size_t i = 0; i < n; ++i) {
      A[(mc + i) * n + i] = 1.0;
      l[mc + i] = std::fmax(lbs_[i], -1e30);
      u[mc + i] = std::fmin(ubs_[i], 1e30);
    }
  }

  CvxOptStatus optimize() override {
    std::size_t n = 0, m = 0;
    DblVec P, q, A, l, u;
    canonicalForm(n, m, P, q, A, l, u);
    tb200_qp_general qp{};
    qp.n = static_cast<int32_t>(n);
    qp.m = static_cast<int32_t>(m);
    qp.batch = 1;
    qp.P = P.data(); qp.q = q.data(); qp.A = A.data(); qp.l = l.data(); qp.u = u.data();
    solution_.assign(n, 0.0);
    duals_.assign(m, 0.0);
    int32_t status = 0, iters = 0, polish = 0;
    const int rc = tb200_qp_solve_general(&qp, &config_.settings, config_.device, solution_.data(), duals_.data(), &status, &iters, &polish);
    if (rc != TB200_OK) throw std::runtime_error(std::string("tb200_qp_solve_general: ") + tb200_qp_general_last_error());
    last_status_ = status;
    last_iters_ = iters;
    // status map of osqp_interface.cpp:565-614
    if (status == 1 || status == 2) return CVX_SOLVED;
    if (status >= 3 && status <= 6) return CVX_INFEASIBLE;
    return CVX_FAILED;
  }
  int lastSolverStatus() const { return last_status_; }
  int lastIterations() const { return last_iters_; }

private:
  Cnt addCnt(const AffExpr& expr, ConstraintType type) {
    const std::scoped_lock lock(mutex_);
    cnts_.emplace_back(std::make_shared<CntRep>(cnts_.size(), this));
    cnts_.back().cnt_rep->type = type;
    cnt_exprs_.push_back(expr);
    cnt_types_.push_back(type);
    return cnts_.back();
  }
  B200ModelConfig config_;
  VarVector vars_;
  CntVector cnts_;
  DblVec lbs_, ubs_, solution_, duals_;
  std::vector<AffExpr> cnt_exprs_;
  std::vector<ConstraintType> cnt_types_;
  QuadExpr objective_;
  std::mutex mutex_;
  int last_status_ = 0, last_iters_ = 0;
};

// solver_interface.hpp:259 / solver_interface.cpp:289-365: every solver name gets the one back end of this library
inline Model::Ptr createModel(ModelType /*model_type*/ = ModelType::AUTO_SOLVER, const ModelConfig::ConstPtr& model_config = nullptr) {
  return std::make_shared<B200Model>(model_config);
}

}  // namespace sco
