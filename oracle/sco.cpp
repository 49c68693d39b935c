// ORACLE — TEST INFRASTRUCTURE ONLY (see sco.hpp header comment).
#include "sco.hpp"
#include <cstdint>
#include <atomic>

#include <algorithm>
#include <cassert>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <numeric>
#include <stdexcept>

namespace oracle {

// ============================================================================ expressions
double AffExpr::value(const double* x) const {
  double out = constant;
  for (size_t i = 0; i < vars.size(); ++i) out += coeffs[i] * x[vars[i]];
  return out;
}
double QuadExpr::value(const double* x) const {  // solver_interface.cpp:92-109
  double out = aff.value(x);
  for (size_t i = 0; i < coeffs.size(); ++i) out += coeffs[i] * x[v1[i]] * x[v2[i]];
  return out;
}
AffExpr cleanupAff(const AffExpr& a) {
  AffExpr out;
  out.constant = a.constant;
  for (size_t i = 0; i < a.vars.size(); ++i)
    if (std::fabs(a.coeffs[i]) > 1e-7) {
      out.vars.push_back(a.vars[i]);
      out.coeffs.push_back(a.coeffs[i]);
    }
  return out;
}
QuadExpr exprSquare(const AffExpr& a) {
  QuadExpr out;
  const size_t k = a.coeffs.size();
  out.aff.constant = a.constant * a.constant;
  out.aff.vars = a.vars;
  out.aff.coeffs.resize(k);
  for (size_t i = 0; i < k; ++i) out.aff.coeffs[i] = 2 * a.constant * a.coeffs[i];
  for (size_t i = 0; i < k; ++i) {
    out.v1.push_back(a.vars[i]);
    out.v2.push_back(a.vars[i]);
    out.coeffs.push_back(a.coeffs[i] * a.coeffs[i]);
    for (size_t j = i + 1; j < k; ++j) {
      out.v1.push_back(a.vars[i]);
      out.v2.push_back(a.vars[j]);
      out.coeffs.push_back(2 * a.coeffs[i] * a.coeffs[j]);
    }
  }
  return out;
}
void exprScale(AffExpr& a, double s) {
  a.constant *= s;
  for (double& c : a.coeffs) c *= s;
}
void exprScale(QuadExpr& q, double s) {
  exprScale(q.aff, s);
  for (double& c : q.coeffs) c *= s;
}
void exprInc(AffExpr& a, const AffExpr& b) {
  a.constant += b.constant;
  a.vars.insert(a.vars.end(), b.vars.begin(), b.vars.end());
  a.coeffs.insert(a.coeffs.end(), b.coeffs.begin(), b.coeffs.end());
}
void exprInc(QuadExpr& a, const AffExpr& b) { exprInc(a.aff, b); }
void exprInc(QuadExpr& a, const QuadExpr& b) {
  exprInc(a.aff, b.aff);
  a.v1.insert(a.v1.end(), b.v1.begin(), b.v1.end());
  a.v2.insert(a.v2.end(), b.v2.begin(), b.v2.end());
  a.coeffs.insert(a.coeffs.end(), b.coeffs.begin(), b.coeffs.end());
}

// ============================================================================ sparse helpers
void Csr::addRow(const std::vector<int>& c, const Vec& v) {
  idx.insert(idx.end(), c.begin(), c.end());
  val.insert(val.end(), v.begin(), v.end());
  ptr.push_back(static_cast<int>(idx.size()));
  ++rows;
}

// Accumulate an affine expression into (sorted, merged, exact-zero-free) index/value lists:
// the doublet sort+merge of solver_utils.cpp:12-47.
static void affToSparse(const AffExpr& e, std::vector<int>& cols, Vec& vals) {
  std::vector<std::pair<int, double>> d;
  d.reserve(e.vars.size());
  for (size_t i = 0; i < e.vars.size(); ++i)
    if (e.coeffs[i] != 0.) d.emplace_back(e.vars[i], e.coeffs[i]);
  std::stable_sort(d.begin(), d.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  cols.clear();
  vals.clear();
  for (const auto& p : d) {
    if (!cols.empty() && cols.back() == p.first)
      vals.back() += p.second;
    else {
      cols.push_back(p.first);
      vals.push_back(p.second);
    }
  }
}
void affToRow(const AffExpr& e, int n_vars, Vec& dense_row) {
  dense_row.assign(n_vars, 0.0);
  std::vector<int> c;
  Vec v;
  affToSparse(e, c, v);
  for (size_t i = 0; i < c.size(); ++i) {
    if (c[i] >= n_vars) throw std::runtime_error("coefficient index beyond n_vars");
    dense_row[c[i]] = v[i];
  }
}

// Quadratic expression -> symmetric matrix entries.  matrix_is_halved: the consumer evaluates
// 1/2 x'Qx, so Q = M + M' with M the upper-triangular coefficient matrix (solver_utils.cpp:70-109).
// Returned as a map keyed by (row<=col) with the FULL symmetric value at (row,col).
static void quadToUpper(const QuadExpr& e, bool halved, bool force_diag, int n,
                        std::vector<std::vector<std::pair<int, double>>>& upper) {
  upper.assign(n, {});
  auto add = [&](int i, int j, double v) {
    if (i > j) std::swap(i, j);
    for (auto& p : upper[i])
      if (p.first == j) {
        p.second += v;
        return;
      }
    upper[i].emplace_back(j, v);
  };
  for (size_t k = 0; k < e.coeffs.size(); ++k) {
    if (e.coeffs[k] == 0.0) continue;
    const int i = e.v1[k], j = e.v2[k];
    if (i == j)
      add(i, i, halved ? 2 * e.coeffs[k] : e.coeffs[k]);
    else  // off-diagonal coefficient c on x_i x_j: symmetric matrix carries c/2 at (i,j) and (j,i)
      add(i, j, halved ? e.coeffs[k] : 0.5 * e.coeffs[k]);
  }
  if (force_diag)
    for (int i = 0; i < n; ++i) add(i, i, 0.0);
  for (auto& r : upper) std::sort(r.begin(), r.end());
}
void quadToDense(const QuadExpr& e, int n, bool halved, bool force_diag, Vec& Q, Vec& q, int& nnz) {
  std::vector<std::vector<std::pair<int, double>>> up;
  quadToUpper(e, halved, force_diag, n, up);
  Q.assign(static_cast<size_t>(n) * n, 0.0);
  nnz = 0;
  for (int i = 0; i < n; ++i)
    for (auto& p : up[i]) {
      Q[i * n + p.first] = p.second;
      Q[p.first * n + i] = p.second;
      nnz += (p.first == i) ? 1 : 2;
    }
  affToRow(e.aff, n, q);
}
void denseToCsc(const Vec& M, int rows, int cols, bool upper_only, std::vector<long long>& row_idx,
                std::vector<long long>& col_ptr, Vec& data) {
  row_idx.clear();
  data.clear();
  col_ptr.assign(1, 0);
  for (int j = 0; j < cols; ++j) {
    for (int i = 0; i < rows; ++i) {
      if (upper_only && i > j) break;
      const double v = M[static_cast<size_t>(i) * cols + j];
      if (v != 0.0) {
        row_idx.push_back(i);
        data.push_back(v);
      }
    }
    col_ptr.push_back(static_cast<long long>(data.size()));
  }
}

// ============================================================================ QP solver
namespace {
constexpr double OSQP_INFTY = 1e30;  // osqp_api_constants.h (v1.0.0) [EXT]
constexpr double MIN_SCALING = 1e-4, MAX_SCALING = 1e4;
constexpr double RHO_MIN = 1e-6, RHO_MAX = 1e6, RHO_TOL = 1e-4, RHO_EQ_OVER_RHO_INEQ = 1e3;

double normInf(const Vec& v) {
  double m = 0;
  for (double e : v) m = std::max(m, std::fabs(e));
  return m;
}
double normInfScaled(const Vec& s, const Vec& v) {
  double m = 0;
  for (size_t i = 0; i < v.size(); ++i) m = std::max(m, std::fabs(s[i] * v[i]));
  return m;
}
void symMatVec(const Csr& Pu, const Vec& x, Vec& y) {
  std::fill(y.begin(), y.end(), 0.0);
  for (int i = 0; i < Pu.rows; ++i)
    for (int k = Pu.ptr[i]; k < Pu.ptr[i + 1]; ++k) {
      const int j = Pu.idx[k];
      y[i] += Pu.val[k] * x[j];
      if (j != i) y[j] += Pu.val[k] * x[i];
    }
}
void matVec(const Csr& A, const Vec& x, Vec& y) {
  for (int i = 0; i < A.rows; ++i) {
    double s = 0;
    for (int k = A.ptr[i]; k < A.ptr[i + 1]; ++k) s += A.val[k] * x[A.idx[k]];
    y[i] = s;
  }
}
void matTVec(const Csr& A, const Vec& y, Vec& x) {
  std::fill(x.begin(), x.end(), 0.0);
  for (int i = 0; i < A.rows; ++i)
    for (int k = A.ptr[i]; k < A.ptr[i + 1]; ++k) x[A.idx[k]] += A.val[k] * y[i];
}
double limitScaling(double v) {
  v = v < MIN_SCALING ? 1.0 : v;
  return v > MAX_SCALING ? MAX_SCALING : v;
}

// Envelope (skyline) Cholesky of a symmetric positive definite matrix under a bandwidth-reducing
// ordering.  Stands in for QDLDL on the quasi-definite KKT system: eliminating nu from
// [[P+sigma I, A'],[A, -diag(1/rho)]] gives (P + sigma I + A' diag(rho) A) x = rhs, the same linear
// map (OSQP's own indirect backend uses exactly this reduced form).
struct EnvChol {
  int n = 0;
  std::vector<int> perm, inv, first, start;
  Vec a;
  double& at(int i, int j) { return a[start[i] + (j - first[i])]; }
  double at(int i, int j) const { return a[start[i] + (j - first[i])]; }

  void analyse(const Csr& Pu, const Csr& A) {
    n = Pu.rows;
    std::vector<std::vector<int>> adj(n);
    auto link = [&](int i, int j) {
      if (i != j) {
        adj[i].push_back(j);
        adj[j].push_back(i);
      }
    };
    for (int i = 0; i < n; ++i)
      for (int k = Pu.ptr[i]; k < Pu.ptr[i + 1]; ++k) link(i, Pu.idx[k]);
    for (int r = 0; r < A.rows; ++r)
      for (int k = A.ptr[r]; k < A.ptr[r + 1]; ++k)
        for (int k2 = k + 1; k2 < A.ptr[r + 1]; ++k2) link(A.idx[k], A.idx[k2]);
    for (auto& v : adj) {
      std::sort(v.begin(), v.end());
      v.erase(std::unique(v.begin(), v.end()), v.end());
    }
    // reverse Cuthill-McKee, components started from a minimum-degree vertex
    std::vector<char> seen(n, 0);
    std::vector<int> order;
    order.reserve(n);
    std::vector<int> by_degree(n);
    std::iota(by_degree.begin(), by_degree.end(), 0);
    std::stable_sort(by_degree.begin(), by_degree.end(),
                     [&](int x, int y) { return adj[x].size() < adj[y].size(); });
    for (int s : by_degree) {
      if (seen[s]) continue;
      size_t head = order.size();
      order.push_back(s);
      seen[s] = 1;
      while (head < order.size()) {
        const int v = order[head++];
        std::vector<int> nb;
        for (int w : adj[v])
          if (!seen[w]) {
            seen[w] = 1;
            nb.push_back(w);
          }
        std::stable_sort(nb.begin(), nb.end(), [&](int x, int y) { return adj[x].size() < adj[y].size(); });
        order.insert(order.end(), nb.begin(), nb.end());
      }
    }
    std::reverse(order.begin(), order.end());
    perm = order;
    inv.assign(n, 0);
    for (int i = 0; i < n; ++i) inv[perm[i]] = i;
    first.assign(n, 0);
    for (int i = 0; i < n; ++i) {
      int f = i;
      for (int w : adj[perm[i]]) f = std::min(f, inv[w]);
      first[i] = f;
    }
    start.assign(n + 1, 0);
    for (int i = 0; i < n; ++i) start[i + 1] = start[i] + (i - first[i] + 1);
    // at(i,j) indexes a[start[i] + j - first[i]]
    a.assign(start[n], 0.0);
  }
  void clear() { std::fill(a.begin(), a.end(), 0.0); }
  void add(int oi, int oj, double v) {  // original indices, symmetric entry
    int i = inv[oi], j = inv[oj];
    if (i < j) std::swap(i, j);
    at(i, j) += v;
  }
  bool factor() {
    for (int i = 0; i < n; ++i) {
      for (int j = first[i]; j < i; ++j) {
        double s = at(i, j);
        const int k0 = std::max(first[i], first[j]);
        for (int k = k0; k < j; ++k) s -= at(i, k) * at(j, k);
        at(i, j) = s / at(j, j);
      }
      double s = at(i, i);
      for (int k = first[i]; k < i; ++k) s -= at(i, k) * at(i, k);
      if (!(s > 0.0)) return false;
      at(i, i) = std::sqrt(s);
    }
    return true;
  }
  void solve(const Vec& b, Vec& x) const {  // original index space
    Vec w(n);
    for (int i = 0; i < n; ++i) w[i] = b[perm[i]];
    for (int i = 0; i < n; ++i) {
      double s = w[i];
      for (int k = first[i]; k < i; ++k) s -= at(i, k) * w[k];
      w[i] = s / at(i, i);
    }
    for (int i = n - 1; i >= 0; --i) {
      w[i] /= at(i, i);
      for (int k = first[i]; k < i; ++k) w[k] -= at(i, k) * w[i];
    }
    for (int i = 0; i < n; ++i) x[perm[i]] = w[i];
  }
};

struct Work {
  int n, m;
  Csr Pu, A;  // scaled data
  Vec q, l, u;
  Vec D, E, Dinv, Einv;
  double c = 1, cinv = 1;
  Vec rho_vec;
  std::vector<int> ctype;  // -1 loose, 0 inequality, 1 equality
  EnvChol K;
  bool assemble(double sigma, const Vec& w) {  // K = P + sigma I + A' diag(w) A
    K.clear();
    for (int i = 0; i < n; ++i) {
      K.add(i, i, sigma);
      for (int k = Pu.ptr[i]; k < Pu.ptr[i + 1]; ++k) K.add(i, Pu.idx[k], Pu.val[k]);
    }
    for (int r = 0; r < m; ++r) {
      if (w[r] == 0.0) continue;
      for (int k = A.ptr[r]; k < A.ptr[r + 1]; ++k)
        for (int k2 = k; k2 < A.ptr[r + 1]; ++k2) K.add(A.idx[k], A.idx[k2], w[r] * A.val[k] * A.val[k2]);
    }
    return K.factor();
  }
};

// scale_data() of OSQP (Ruiz equilibration of the KKT matrix + cost normalisation) [EXT]
void ruizScale(Work& w, int passes) {
  const int n = w.n, m = w.m;
  w.D.assign(n, 1.0);
  w.E.assign(m, 1.0);
  w.c = 1.0;
  Vec Dt(n), Et(m);
  for (int it = 0; it < passes; ++it) {
    std::fill(Dt.begin(), Dt.end(), 0.0);
    std::fill(Et.begin(), Et.end(), 0.0);
    for (int i = 0; i < n; ++i)
      for (int k = w.Pu.ptr[i]; k < w.Pu.ptr[i + 1]; ++k) {
        const double v = std::fabs(w.Pu.val[k]);
        Dt[i] = std::max(Dt[i], v);
        Dt[w.Pu.idx[k]] = std::max(Dt[w.Pu.idx[k]], v);
      }
    for (int r = 0; r < m; ++r)
      for (int k = w.A.ptr[r]; k < w.A.ptr[r + 1]; ++k) {
        const double v = std::fabs(w.A.val[k]);
        Dt[w.A.idx[k]] = std::max(Dt[w.A.idx[k]], v);
        Et[r] = std::max(Et[r], v);
      }
    for (double& d : Dt) d = 1.0 / std::sqrt(limitScaling(d));
    for (double& e : Et) e = 1.0 / std::sqrt(limitScaling(e));
    for (int i = 0; i < n; ++i)
      for (int k = w.Pu.ptr[i]; k < w.Pu.ptr[i + 1]; ++k) w.Pu.val[k] *= Dt[i] * Dt[w.Pu.idx[k]];
    for (int r = 0; r < m; ++r)
      for (int k = w.A.ptr[r]; k < w.A.ptr[r + 1]; ++k) w.A.val[k] *= Et[r] * Dt[w.A.idx[k]];
    for (int i = 0; i < n; ++i) {
      w.q[i] *= Dt[i];
      w.D[i] *= Dt[i];
    }
    for (int r = 0; r < m; ++r) w.E[r] *= Et[r];
    // cost normalisation: mean column inf-norm of P vs inf-norm of q
    Vec cn(n, 0.0);
    for (int i = 0; i < n; ++i)
      for (int k = w.Pu.ptr[i]; k < w.Pu.ptr[i + 1]; ++k) {
        const double v = std::fabs(w.Pu.val[k]);
        cn[i] = std::max(cn[i], v);
        cn[w.Pu.idx[k]] = std::max(cn[w.Pu.idx[k]], v);
      }
    double mean = 0;
    for (double v : cn) mean += v;
    mean = limitScaling(mean / n);
    const double qn = limitScaling(normInf(w.q));
    const double ct = 1.0 / std::max(mean, qn);
    for (double& v : w.Pu.val) v *= ct;
    for (double& v : w.q) v *= ct;
    w.c *= ct;
  }
  w.Dinv.resize(n);
  w.Einv.resize(m);
  for (int i = 0; i < n; ++i) w.Dinv[i] = 1.0 / w.D[i];
  for (int r = 0; r < m; ++r) w.Einv[r] = 1.0 / w.E[r];
  w.cinv = 1.0 / w.c;
  for (int r = 0; r < m; ++r) {
    w.l[r] *= w.E[r];
    w.u[r] *= w.E[r];
  }
}

void setRhoValues(Work& w, double rho) {
  for (int r = 0; r < w.m; ++r)
    if (w.ctype[r] == 0) w.rho_vec[r] = rho;
    else if (w.ctype[r] == 1) w.rho_vec[r] = RHO_EQ_OVER_RHO_INEQ * rho;
}
void setRhoVec(Work& w, double rho) {
  w.rho_vec.resize(w.m);
  w.ctype.resize(w.m);
  for (int r = 0; r < w.m; ++r) {
    if (w.l[r] < -OSQP_INFTY * MIN_SCALING && w.u[r] > OSQP_INFTY * MIN_SCALING) {
      w.ctype[r] = -1;
      w.rho_vec[r] = RHO_MIN;
    } else if (w.u[r] - w.l[r] < RHO_TOL) {
      w.ctype[r] = 1;
      w.rho_vec[r] = RHO_EQ_OVER_RHO_INEQ * rho;
    } else {
      w.ctype[r] = 0;
      w.rho_vec[r] = rho;
    }
  }
}
}  // namespace

// splitmix64 finaliser: the per-row term of the active-set hash of optimisation O1
static inline uint64_t guess_mix(uint64_t v) {
  v += 0x9e3779b97f4a7c15ull;
  v = (v ^ (v >> 30)) * 0xbf58476d1ce4e5b9ull;
  v = (v ^ (v >> 27)) * 0x94d049bb133111ebull;
  return v ^ (v >> 31);
}

QPResult qp_solve(const QP& qp, const QPSettings& s, const QPWarmStart* warm) {
  const int n = qp.n, m = qp.m;
  Work w;
  w.n = n;
  w.m = m;
  w.Pu = qp.Pu;
  w.A = qp.A;
  w.q = qp.q;
  w.l = qp.l;
  w.u = qp.u;
  // bounds beyond OSQP_INFTY (+-inf included) mean "none": clamp them as the device kernels do, so that no inf
  // reaches a product (inf * 0 = NaN in the polish right-hand side and the infeasibility certificate)
  for (int r = 0; r < m; ++r) {
    w.l[r] = std::max(w.l[r], -OSQP_INFTY);
    w.u[r] = std::min(w.u[r], OSQP_INFTY);
  }
  if (s.scaling > 0)
    ruizScale(w, s.scaling);
  else {
    w.D.assign(n, 1.0);
    w.Dinv = w.D;
    w.E.assign(m, 1.0);
    w.Einv = w.E;
  }
  double rho = (warm && warm->valid) ? warm->rho : s.rho;
  rho = std::min(std::max(rho, RHO_MIN), RHO_MAX);
  setRhoVec(w, rho);
  w.K.analyse(w.Pu, w.A);

  QPResult res;
  res.x.assign(n, 0.0);
  res.y.assign(m, 0.0);
  if (!w.assemble(s.sigma, w.rho_vec)) {
    res.status = QP_NON_CVX;
    return res;
  }

  Vec x(n, 0.0), z(m, 0.0), y(m, 0.0), xp(n), zp(m), xt(n), zt(m), rhs(n), tmp_m(m), tmp_n(n);
  Vec Ax(m), Px(n), Aty(n), dx(n), dy(m);
  if (warm && warm->valid && static_cast<int>(warm->x.size()) == n && static_cast<int>(warm->y.size()) == m) {
    // osqp_warm_start: x <- Dinv x, y <- c Einv y, z <- A x   [EXT]
    for (int i = 0; i < n; ++i) x[i] = warm->x[i] * w.Dinv[i];
    for (int r = 0; r < m; ++r) y[r] = warm->y[r] * w.Einv[r] * w.c;
    matVec(w.A, x, z);
  }

  double pri_res = 0, dua_res = 0;
  auto updateInfo = [&]() {
    matVec(w.A, x, Ax);
    symMatVec(w.Pu, x, Px);
    matTVec(w.A, y, Aty);
    double p = 0;
    for (int r = 0; r < m; ++r) p = std::max(p, std::fabs(w.Einv[r] * (Ax[r] - z[r])));
    pri_res = p;
    double d = 0;
    for (int i = 0; i < n; ++i) d = std::max(d, std::fabs(w.Dinv[i] * (w.q[i] + Px[i] + Aty[i])));
    dua_res = d * w.cinv;
  };
  auto primalInfeasible = [&](double eps) {
    Vec d = dy;
    for (int r = 0; r < m; ++r) {
      if (w.u[r] > OSQP_INFTY * MIN_SCALING) {
        if (w.l[r] < -OSQP_INFTY * MIN_SCALING)
          d[r] = 0.0;
        else
          d[r] = std::min(d[r], 0.0);
      } else if (w.l[r] < -OSQP_INFTY * MIN_SCALING) {
        d[r] = std::max(d[r], 0.0);
      }
    }
    const double nd = normInfScaled(w.E, d);
    if (nd > eps) {
      double lhs = 0;
      for (int r = 0; r < m; ++r) lhs += w.u[r] * std::max(d[r], 0.0) + w.l[r] * std::min(d[r], 0.0);
      if (lhs < -eps * nd) {
        matTVec(w.A, d, tmp_n);
        return normInfScaled(w.Dinv, tmp_n) < eps * nd;
      }
    }
    return false;
  };
  auto dualInfeasible = [&](double eps) {
    const double ndx = normInfScaled(w.D, dx);
    if (ndx > eps) {
      double qdx = 0;
      for (int i = 0; i < n; ++i) qdx += w.q[i] * dx[i];
      if (qdx < -w.c * eps * ndx) {
        symMatVec(w.Pu, dx, tmp_n);
        if (normInfScaled(w.Dinv, tmp_n) < w.c * eps * ndx) {
          matVec(w.A, dx, tmp_m);
          for (int r = 0; r < m; ++r) {
            const double v = w.Einv[r] * tmp_m[r];
            if ((w.u[r] < OSQP_INFTY * MIN_SCALING && v > eps * ndx) ||
                (w.l[r] > -OSQP_INFTY * MIN_SCALING && v < -eps * ndx))
              return false;
          }
          return true;
        }
      }
    }
    return false;
  };
  // check_termination() of OSQP [EXT]; returns status or QP_UNSOLVED
  double eps_scale = 1.0;  // tightened by the verified-polish rounds (deviation D2)
  auto checkTermination = [&](bool approximate) -> int {
    double eps_abs = s.eps_abs * eps_scale, eps_rel = s.eps_rel * eps_scale, epi = s.eps_prim_inf, edi = s.eps_dual_inf;
    if (approximate) {
      eps_abs *= 10;
      eps_rel *= 10;
      epi *= 10;
      edi *= 10;
    }
    if (pri_res > OSQP_INFTY || dua_res > OSQP_INFTY) return QP_NON_CVX;
    const double eps_pri = eps_abs + eps_rel * std::max(normInfScaled(w.Einv, z), normInfScaled(w.Einv, Ax));
    const double eps_dua =
        eps_abs + eps_rel * w.cinv *
                      std::max(normInfScaled(w.Dinv, w.q), std::max(normInfScaled(w.Dinv, Aty), normInfScaled(w.Dinv, Px)));
    bool pri_ok = pri_res < eps_pri, dua_ok = dua_res < eps_dua, pinf = false, dinf = false;
    if (!pri_ok) pinf = primalInfeasible(epi);
    if (!dua_ok) dinf = dualInfeasible(edi);
    if (pri_ok && dua_ok) return approximate ? QP_SOLVED_INACCURATE : QP_SOLVED;
    if (pinf) return approximate ? QP_PRIMAL_INFEASIBLE_INACCURATE : QP_PRIMAL_INFEASIBLE;
    if (dinf) return approximate ? QP_DUAL_INFEASIBLE_INACCURATE : QP_DUAL_INFEASIBLE;
    return QP_UNSOLVED;
  };

  int status = QP_UNSOLVED, iter = 0;
  bool early_verified = false;
  std::function<bool(bool&)> polishOnce;
  // hash of the active-set guess the polish would start from (order independent sum, wraps mod 2^64)
  uint64_t prev_guess = 0, failed_guess = 0, pending_guess = 0;
  bool have_prev_guess = false, have_failed_guess = false;
  auto guessHash = [&]() -> uint64_t {
    uint64_t h = 0;
    for (int r = 0; r < m; ++r) {
      int a = 0;
      if (z[r] - w.l[r] < -y[r]) a = -1;
      else if (w.u[r] - z[r] < y[r]) a = 1;
      if (a) h += guess_mix(2 * static_cast<uint64_t>(r) + (a > 0 ? 1 : 0));
    }
    return h;
  };
  // ADMM iterations, continuing from the current state until a termination test fires or max_iter.
  auto runAdmm = [&]() {
    status = QP_UNSOLVED;
    while (iter < s.max_iter) {
      ++iter;
      xp = x;
      zp = z;
      // update_xz_tilde: (P + sigma I + A' R A) xt = sigma x_prev - q + A'(R z_prev - y);  zt = A xt
      for (int r = 0; r < m; ++r) tmp_m[r] = w.rho_vec[r] * zp[r] - y[r];
      matTVec(w.A, tmp_m, rhs);
      for (int i = 0; i < n; ++i) rhs[i] += s.sigma * xp[i] - w.q[i];
      w.K.solve(rhs, xt);
      matVec(w.A, xt, zt);
      for (int i = 0; i < n; ++i) {
        x[i] = s.alpha * xt[i] + (1 - s.alpha) * xp[i];
        dx[i] = x[i] - xp[i];
      }
      for (int r = 0; r < m; ++r) {
        const double zr = s.alpha * zt[r] + (1 - s.alpha) * zp[r];
        double v = zr + y[r] / w.rho_vec[r];
        v = std::min(std::max(v, w.l[r]), w.u[r]);
        z[r] = v;
        dy[r] = w.rho_vec[r] * (zr - v);
        y[r] += dy[r];
      }
      const bool can_check = s.check_termination > 0 && (iter % s.check_termination == 0);
      if (can_check) {
        updateInfo();
        status = checkTermination(false);
        if (status != QP_UNSOLVED) return;
        // the early polish is a polish: without polishing, ADMM alone must meet its tolerances (as in both kernels)
        bool try_early = s.polishing && s.early_polish_every > 0 && iter >= s.early_polish_from &&
                         (iter % s.early_polish_every == 0);
        if (try_early && s.early_polish_stable) {
          // only when the active-set guess has settled (same as at the previous test) and has not failed before
          const uint64_t h = guessHash();
          const bool stable = have_prev_guess && h == prev_guess;
          prev_guess = h;
          have_prev_guess = true;
          try_early = stable && !(have_failed_guess && h == failed_guess);
          if (try_early) pending_guess = h;
        }
        if (try_early) {
          // optimisation O1: try the polish before ADMM has met its own tolerances; a VERIFIED polished point is
          // the exact minimiser no matter how rough the iterate that produced the active-set guess was
          bool verified = false;
          const double keep_pri = pri_res, keep_dua = dua_res;
          const bool factored = polishOnce(verified);
          ++res.early_tries;
          if (getenv("ORACLE_COUNT_TRIES")) { static std::atomic<long> n{0}; long v = ++n; if (v % 1000 == 0) fprintf(stderr, "early tries so far %ld\n", v); }
          if (factored && verified) {
            early_verified = true;
            status = QP_SOLVED;
            return;
          }
          (void)keep_pri;
          (void)keep_dua;
          failed_guess = pending_guess;
          have_failed_guess = true;
          updateInfo();  // the polish scratch vectors are shared with the residual bookkeeping
          if (!w.assemble(s.sigma, w.rho_vec)) {
            status = QP_NON_CVX;
            return;
          }
        }
      }
      if (s.adaptive_rho && s.adaptive_rho_interval > 0 && (iter % s.adaptive_rho_interval == 0)) {
        if (!can_check) updateInfo();
        // compute_rho_estimate (scaled quantities) [EXT]
        double p = 0, d = 0;
        for (int r = 0; r < m; ++r) p = std::max(p, std::fabs(Ax[r] - z[r]));
        for (int i = 0; i < n; ++i) d = std::max(d, std::fabs(w.q[i] + Px[i] + Aty[i]));
        p /= (std::max(normInf(z), normInf(Ax)) + 1e-10);
        d /= (std::max(normInf(w.q), std::max(normInf(Aty), normInf(Px))) + 1e-10);
        double rho_new = rho * std::sqrt(p / (d + 1e-10));
        rho_new = std::min(std::max(rho_new, RHO_MIN), RHO_MAX);
        if (rho_new > rho * s.adaptive_rho_tolerance || rho_new < rho / s.adaptive_rho_tolerance) {
          rho = rho_new;
          setRhoValues(w, rho);
          if (!w.assemble(s.sigma, w.rho_vec)) {
            status = QP_NON_CVX;
            return;
          }
          ++res.rho_updates;
        }
      }
    }
    // max_iter reached without a verdict: approximate test, then MAX_ITER_REACHED
    if (!(s.check_termination > 0 && (iter % s.check_termination == 0))) updateInfo();
    status = checkTermination(true);
    if (status == QP_UNSOLVED) status = QP_MAX_ITER_REACHED;
  };

  // ---- polish (OSQP polish.c [EXT]): equality-constrained QP on the guessed active set, solved as the
  // delta-regularised KKT system + iterative refinement, written in its reduced (proximal method of
  // multipliers) form  K_p = P + delta I + (1/delta) A_act' A_act.
  // DEVIATION D2 (DESIGN.md): OSQP polishes once and keeps the result whenever its residuals beat ADMM's, even
  // when the guessed active set was wrong (the point is then NOT the QP minimiser and depends on the ADMM
  // path).  Here a polished point is accepted at once only when it is VERIFIED: primal feasible to verify_tol
  // and with correctly signed multipliers on its active inequality rows, i.e. a KKT point = the unique
  // minimiser, independent of how the guess was produced.  Otherwise ADMM continues from where it stopped
  // with 10x tighter tolerances and the polish is retried (verify_rounds times); only then OSQP's own
  // acceptance rule is used.  verify_rounds = 0 is plain OSQP behaviour.
  Vec wact(m), b(m), xq(n), yq(m), rd(n), step(n);
  double pp = 0, pdres = 0;
  polishOnce = [&](bool& verified) -> bool {
    verified = false;
    for (int r = 0; r < m; ++r) {
      int a = 0;
      if (z[r] - w.l[r] < -y[r]) a = -1;
      else if (w.u[r] - z[r] < y[r]) a = 1;
      wact[r] = a ? 1.0 / s.delta : 0.0;
      b[r] = a < 0 ? w.l[r] : w.u[r];
      tmp_m[r] = a;
    }
    Vec act = tmp_m;
    if (!w.assemble(s.delta, wact)) return false;
    std::fill(xq.begin(), xq.end(), 0.0);
    std::fill(yq.begin(), yq.end(), 0.0);
    for (int it = 0; it <= s.polish_refine_iter; ++it) {
      symMatVec(w.Pu, xq, Px);
      matTVec(w.A, yq, Aty);
      matVec(w.A, xq, Ax);
      for (int r = 0; r < m; ++r) tmp_m[r] = wact[r] * (Ax[r] - b[r]);
      matTVec(w.A, tmp_m, tmp_n);
      for (int i = 0; i < n; ++i) rd[i] = -(Px[i] + w.q[i] + Aty[i]) - tmp_n[i];
      w.K.solve(rd, step);
      for (int i = 0; i < n; ++i) xq[i] += step[i];
      matVec(w.A, xq, Ax);
      for (int r = 0; r < m; ++r)
        if (wact[r] != 0.0) yq[r] += wact[r] * (Ax[r] - b[r]);
    }
    matVec(w.A, xq, Ax);
    symMatVec(w.Pu, xq, Px);
    matTVec(w.A, yq, Aty);
    pp = pdres = 0;
    bool signs_ok = true;
    for (int r = 0; r < m; ++r) {
      const double zr = std::min(std::max(Ax[r], w.l[r]), w.u[r]);
      pp = std::max(pp, std::fabs(w.Einv[r] * (Ax[r] - zr)));
      if (act[r] != 0 && w.u[r] - w.l[r] >= RHO_TOL) {  // inequality row held active: multiplier sign
        if (act[r] > 0 && yq[r] < -s.verify_tol) signs_ok = false;
        if (act[r] < 0 && yq[r] > s.verify_tol) signs_ok = false;
      }
    }
    for (int i = 0; i < n; ++i) pdres = std::max(pdres, std::fabs(w.Dinv[i] * (w.q[i] + Px[i] + Aty[i])));
    pdres *= w.cinv;
    verified = signs_ok && pp <= s.verify_tol && std::isfinite(pp) && std::isfinite(pdres);
    return true;
  };

  int round = 0;
  double admm_pri = 0, admm_dua = 0;
  while (true) {
    runAdmm();
    admm_pri = pri_res;
    admm_dua = dua_res;
    if (status != QP_SOLVED || !s.polishing) break;
    if (early_verified) {
      res.polish = 1;
      break;
    }
    bool verified = false;
    const bool factored = polishOnce(verified);
    res.pdas = round;
    if (factored && verified) {
      res.polish = 1;
      break;
    }
    if (round >= s.verify_rounds || iter >= s.max_iter) {  // OSQP's acceptance rule
      const bool ok = factored && ((pp < pri_res && pdres < dua_res) || (pp < pri_res && dua_res < 1e-10) ||
                                   (pdres < dua_res && pri_res < 1e-10)) && std::isfinite(pp) && std::isfinite(pdres);
      res.polish = ok ? 2 : -1;
      break;
    }
    ++round;
    eps_scale *= 0.1;
    if (!w.assemble(s.sigma, w.rho_vec)) {  // back to the ADMM factor
      status = QP_NON_CVX;
      break;
    }
  }
  res.iters = iter;
  res.status = status;
  res.rho = rho;
  res.pri_res = pri_res;
  res.dua_res = dua_res;
  res.admm_pri = admm_pri;
  res.admm_dua = admm_dua;
  res.warm = (warm && warm->valid) ? 1 : 0;
  res.y_admm.assign(m, 0.0);
  for (int r = 0; r < m; ++r) res.y_admm[r] = w.cinv * w.E[r] * y[r];
  if (res.polish > 0) {
    x = xq;
    y = yq;
    res.pri_res = pp;
    res.dua_res = pdres;
  }
  for (int i = 0; i < n; ++i) res.x[i] = w.D[i] * x[i];
  for (int r = 0; r < m; ++r) res.y[r] = w.cinv * w.E[r] * y[r];
  if (getenv("ORACLE_QP_DEBUG"))
    fprintf(stderr, "QP n=%d m=%d status=%d iters=%d rho_upd=%d polish=%d pdas=%d admm_pri=%.2e admm_dua=%.2e pri=%.2e dua=%.2e warm=%d\n", n, m,
            status, res.iters, res.rho_updates, res.polish, res.pdas, admm_pri, admm_dua, res.pri_res, res.dua_res, (int)(warm && warm->valid));
  return res;
}

void qp_kkt_residuals(const QP& qp, const Vec& x, const Vec& y, double& stat, double& prim, double& comp) {
  Vec Px(qp.n), Aty(qp.n), Ax(qp.m);
  symMatVec(qp.Pu, x, Px);
  matTVec(qp.A, y, Aty);
  matVec(qp.A, x, Ax);
  stat = prim = comp = 0;
  for (int i = 0; i < qp.n; ++i) stat = std::max(stat, std::fabs(Px[i] + qp.q[i] + Aty[i]));
  for (int r = 0; r < qp.m; ++r) {
    prim = std::max(prim, std::max(qp.l[r] - Ax[r], Ax[r] - qp.u[r]));
    // y+ acts on the upper bound, y- on the lower bound
    const double up = std::max(y[r], 0.0), lo = std::min(y[r], 0.0);
    if (qp.u[r] < 1e29) comp = std::max(comp, std::fabs(up * (qp.u[r] - Ax[r])));
    else comp = std::max(comp, up);
    if (qp.l[r] > -1e29) comp = std::max(comp, std::fabs(lo * (Ax[r] - qp.l[r])));
    else comp = std::max(comp, -lo);
  }
  prim = std::max(prim, 0.0);
}

// ============================================================================ model
int Model::addVar(double lb, double ub) {
  lbs_.push_back(lb);
  ubs_.push_back(ub);
  return numVars() - 1;
}
void Model::truncateToPermanent() {
  lbs_.resize(n_perm_vars_);
  ubs_.resize(n_perm_vars_);
  cnt_exprs_.resize(n_perm_cnts_);
  cnt_types_.resize(n_perm_cnts_);
}
void Model::buildQP(QP& qp) const {
  const int n = numVars(), mc = numCnts();
  qp.n = n;
  qp.m = mc + n;
  // P = M + M' (upper triangle), q = linear part: updateObjective, osqp_interface.cpp:170-211
  std::vector<std::vector<std::pair<int, double>>> up;
  quadToUpper(objective_, true, false, n, up);
  qp.Pu = Csr();
  qp.Pu.rows = 0;
  qp.Pu.cols = n;
  for (int i = 0; i < n; ++i) {
    std::vector<int> c;
    Vec v;
    for (auto& p : up[i]) {
      c.push_back(p.first);
      v.push_back(p.second);
    }
    qp.Pu.addRow(c, v);
  }
  affToRow(objective_.aff, n, qp.q);
  // A = [cnt rows; I], l/u: updateConstraints, osqp_interface.cpp:213-281
  qp.A = Csr();
  qp.A.cols = n;
  qp.l.assign(qp.m, -OSQP_INFTY);
  qp.u.assign(qp.m, OSQP_INFTY);
  std::vector<int> c;
  Vec v;
  for (int r = 0; r < mc; ++r) {
    affToSparse(cnt_exprs_[r], c, v);
    qp.A.addRow(c, v);
    const double rhs = -cnt_exprs_[r].constant;
    qp.l[r] = cnt_types_[r] == INEQ ? -OSQP_INFTY : rhs;
    qp.u[r] = rhs;
  }
  for (int i = 0; i < n; ++i) {
    qp.A.addRow({i}, {1.0});
    qp.l[mc + i] = std::fmax(lbs_[i], -OSQP_INFTY);
    qp.u[mc + i] = std::fmin(ubs_[i], OSQP_INFTY);
  }
}
CvxStatus Model::optimize() {
  QP qp;
  buildQP(qp);
  // createOrUpdateSolver (osqp_interface.cpp:283-370): with update_workspace == false the workspace is
  // rebuilt every call; an explicit warm start (previous x, y and rho) is applied when the previous
  // solve succeeded and the sparsity of P and A is unchanged.  The reference compares the CSC index
  // arrays with memcmp over n+1 / nnz BYTES (not elements), i.e. effectively dimensions + nnz; the
  // restatement compares (n, m, nnz(P), nnz(A)).
  QPWarmStart ws;
  const bool same = have_last_ && qp.n == last_n_ && qp.m == last_m_ && qp.Pu.nnz() == last_nnzP_ &&
                    qp.A.nnz() == last_nnzA_;
  if (same && settings_.warm_starting && (last_.status == QP_SOLVED || last_.status == QP_SOLVED_INACCURATE)) {
    ws.valid = true;
    ws.x = last_.x;
    // DEVIATION (documented in DESIGN.md): the reference warm-starts from OSQP's returned duals, which are
    // the POLISHED duals when polish succeeded.  On degenerate active sets (linearly dependent bounds + rows,
    // common at trust-box corners) those are non-unique and only fixed by the 1e-6 regularisation, i.e. not
    // reproducible across linear-algebra back ends.  Primal x from polish, duals from the last ADMM iterate.
    ws.y = settings_.warm_polished_duals ? last_.y : last_.y_admm;
    ws.rho = last_.rho;
  }
  last_ = qp_solve(qp, settings_, ws.valid ? &ws : nullptr);
  have_last_ = true;
  last_n_ = qp.n;
  last_m_ = qp.m;
  last_nnzP_ = qp.Pu.nnz();
  last_nnzA_ = qp.A.nnz();
  total_iters_ += last_.iters;
  solution_ = last_.x;
  switch (last_.status) {  // osqp_interface.cpp:565-614
    case QP_SOLVED:
    case QP_SOLVED_INACCURATE:
      return CVX_SOLVED;
    case QP_PRIMAL_INFEASIBLE:
    case QP_PRIMAL_INFEASIBLE_INACCURATE:
    case QP_DUAL_INFEASIBLE:
    case QP_DUAL_INFEASIBLE_INACCURATE:
      return CVX_INFEASIBLE;
    default:
      return CVX_FAILED;
  }
}

// ============================================================================ convex pieces
void ConvexObjective::addHinge(const AffExpr& a, double coeff) {
  const int h = model->addVar(0, kInf);
  AffExpr row = a;
  row.vars.push_back(h);
  row.coeffs.push_back(-1.0);
  ineqs.push_back(row);
  AffExpr cost = AffExpr::var(h);
  exprScale(cost, coeff);
  exprInc(quad, cost);
}
void ConvexObjective::addAbs(const AffExpr& a, double coeff) {
  const int neg = model->addVar(0, kInf);
  const int pos = model->addVar(0, kInf);
  AffExpr cost;
  cost.vars = {neg, pos};
  cost.coeffs = {coeff, coeff};
  exprInc(quad, cost);
  AffExpr row = a;
  row.vars.push_back(neg);
  row.coeffs.push_back(1.0);
  row.vars.push_back(pos);
  row.coeffs.push_back(-1.0);
  eqs.push_back(row);
}
void ConvexObjective::addConstraintsToModel() {
  for (const AffExpr& e : eqs) model->addEqCnt(e);
  for (const AffExpr& e : ineqs) model->addIneqCnt(e);
}
Vec ConvexConstraints::violations(const double* x) const {
  Vec out;
  for (const AffExpr& e : eqs) out.push_back(std::fabs(e.value(x)));
  for (const AffExpr& e : ineqs) out.push_back(std::max(e.value(x), 0.0));
  return out;
}
double ConvexConstraints::violation(const double* x) const {
  double s = 0;
  for (double v : violations(x)) s += v;
  return s;
}
Vec Constraint::violations(const Vec& x) {
  Vec val = value(x);
  for (double& v : val) v = (type() == EQ) ? std::fabs(v) : std::max(v, 0.0);
  return val;
}
double Constraint::violation(const Vec& x) {
  double s = 0;
  for (double v : violations(x)) s += v;
  return s;
}

std::vector<int> OptProb::createVariables(int count, const Vec& lb, const Vec& ub) {
  std::vector<int> out;
  for (int i = 0; i < count; ++i) {
    out.push_back(model_->addVar(lb[i], ub[i]));
    lb_.push_back(lb[i]);
    ub_.push_back(ub[i]);
  }
  model_->markPermanent();
  return out;
}
std::vector<int> OptProb::createVariables(int count) {
  return createVariables(count, Vec(count, -kInf), Vec(count, kInf));
}
void OptProb::addConstraint(std::shared_ptr<Constraint> c) {
  if (c->type() == EQ)
    eqcnts_.push_back(std::move(c));
  else
    ineqcnts_.push_back(std::move(c));
}
void OptProb::addLinearConstraint(const AffExpr& e, CntType t) {
  if (t == EQ)
    model_->addEqCnt(e);
  else
    model_->addIneqCnt(e);
  model_->markPermanent();
}
std::vector<std::shared_ptr<Constraint>> OptProb::getConstraints() const {
  std::vector<std::shared_ptr<Constraint>> out(eqcnts_);
  out.insert(out.end(), ineqcnts_.begin(), ineqcnts_.end());
  return out;
}
Vec OptProb::getClosestFeasiblePoint(const Vec& x, double delta) const {
  Vec y(x.size());
  for (size_t i = 0; i < x.size(); ++i) {
    y[i] = std::fmax(lb_[i] + delta, x[i]);
    y[i] = std::fmin(ub_[i] - delta, x[i]);  // overwrites the lower clip, as the reference does
  }
  return y;
}

// ============================================================================ func wrapping
static Vec gather(const Vec& x, const std::vector<int>& vars) {
  Vec out(vars.size());
  for (size_t i = 0; i < vars.size(); ++i) out[i] = x[vars[i]];
  return out;
}
static AffExpr affFromValGrad(double y, const Vec& x, const Vec& dydx, const std::vector<int>& vars) {
  AffExpr aff;  // modeling_utils.cpp:31-39
  double dot = 0;
  for (size_t i = 0; i < x.size(); ++i) dot += dydx[i] * x[i];
  aff.constant = y - dot;
  aff.coeffs = dydx;
  aff.vars = vars;
  return cleanupAff(aff);
}
std::vector<Vec> calcForwardNumJac(const VectorFn& f, const Vec& x, double eps) {
  const Vec y = f(x);
  std::vector<Vec> J(y.size(), Vec(x.size()));
  Vec xp = x;
  for (size_t i = 0; i < x.size(); ++i) {
    xp[i] = x[i] + eps;
    const Vec yp = f(xp);
    for (size_t r = 0; r < y.size(); ++r) J[r][i] = (yp[r] - y[r]) / eps;
    xp[i] = x[i];
  }
  return J;
}
static Vec calcForwardNumGrad(const ScalarFn& f, const Vec& x, double eps) {  // num_diff.cpp:40-54
  Vec out(x.size()), xp = x;
  const double y = f(x);
  for (size_t i = 0; i < x.size(); ++i) {
    xp[i] = x[i] + eps;
    out[i] = (f(xp) - y) / eps;
    xp[i] = x[i];
  }
  return out;
}
// Jacobi eigen-decomposition of a small symmetric matrix (stands in for Eigen::SelfAdjointEigenSolver
// in modeling_utils.cpp:84-92).
static void symEig(std::vector<Vec> A, Vec& evals, std::vector<Vec>& evecs) {
  const int n = static_cast<int>(A.size());
  evecs.assign(n, Vec(n, 0.0));
  for (int i = 0; i < n; ++i) evecs[i][i] = 1.0;
  for (int sweep = 0; sweep < 100; ++sweep) {
    double off = 0;
    for (int i = 0; i < n; ++i)
      for (int j = i + 1; j < n; ++j) off += A[i][j] * A[i][j];
    if (off < 1e-30) break;
    for (int p = 0; p < n; ++p)
      for (int q = p + 1; q < n; ++q) {
        if (std::fabs(A[p][q]) < 1e-300) continue;
        const double theta = (A[q][q] - A[p][p]) / (2 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        const double c = 1 / std::sqrt(t * t + 1), sn = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - sn * akq;
          A[k][q] = sn * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - sn * aqk;
          A[q][k] = sn * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = evecs[k][p], vkq = evecs[k][q];
          evecs[k][p] = c * vkp - sn * vkq;
          evecs[k][q] = sn * vkp + c * vkq;
        }
      }
  }
  evals.resize(n);
  for (int i = 0; i < n; ++i) evals[i] = A[i][i];
}

double CostFromFunc::value(const Vec& x) { return f_(gather(x, vars_)); }
std::shared_ptr<ConvexObjective> CostFromFunc::convex(const Vec& xall, Model* model) {
  const Vec x = gather(xall, vars_);
  const int n = static_cast<int>(x.size());
  auto out = std::make_shared<ConvexObjective>(model);
  QuadExpr& quad = out->quad;
  if (!full_hessian_) {  // calcGradAndDiagHess, num_diff.cpp:70-91
    const double y = f_(x);
    Vec grad(n), hess(n), xp = x;
    for (int i = 0; i < n; ++i) {
      xp[i] = x[i] + epsilon_ / 2;
      const double yp = f_(xp);
      xp[i] = x[i] - epsilon_ / 2;
      const double ym = f_(xp);
      grad[i] = (yp - ym) / epsilon_;
      hess[i] = std::max((yp + ym - 2 * y) / (epsilon_ * epsilon_ / 4), 0.0);
      xp[i] = x[i];
    }
    double gx = 0, xhx = 0;
    for (int i = 0; i < n; ++i) {
      gx += grad[i] * x[i];
      xhx += x[i] * hess[i] * x[i];
    }
    quad.aff.constant = y - gx + .5 * xhx;
    quad.aff.vars = vars_;
    quad.aff.coeffs.resize(n);
    for (int i = 0; i < n; ++i) quad.aff.coeffs[i] = grad[i] - hess[i] * x[i];
    quad.v1 = vars_;
    quad.v2 = vars_;
    quad.coeffs.resize(n);
    for (int i = 0; i < n; ++i) quad.coeffs[i] = hess[i] * .5;
  } else {  // calcGradHess, num_diff.cpp:93-105 + PSD projection, modeling_utils.cpp:76-112
    const double y = f_(x);
    const Vec grad = calcForwardNumGrad(f_, x, epsilon_);
    VectorFn gfn = [&](const Vec& v) { return calcForwardNumGrad(f_, v, epsilon_); };
    std::vector<Vec> H = calcForwardNumJac(gfn, x, epsilon_);
    for (int i = 0; i < n; ++i)
      for (int j = i + 1; j < n; ++j) H[i][j] = H[j][i] = (H[i][j] + H[j][i]) / 2;
    Vec ev;
    std::vector<Vec> V;
    symEig(H, ev, V);
    std::vector<Vec> Hp(n, Vec(n, 0.0));
    for (int k = 0; k < n; ++k)
      if (ev[k] > 0)
        for (int i = 0; i < n; ++i)
          for (int j = 0; j < n; ++j) Hp[i][j] += ev[k] * V[i][k] * V[j][k];
    double gx = 0, xhx = 0;
    Vec hx(n, 0.0);
    for (int i = 0; i < n; ++i) {
      gx += grad[i] * x[i];
      for (int j = 0; j < n; ++j) hx[i] += Hp[i][j] * x[j];
    }
    for (int i = 0; i < n; ++i) xhx += x[i] * hx[i];
    quad.aff.constant = y - gx + .5 * xhx;
    quad.aff.vars = vars_;
    quad.aff.coeffs.resize(n);
    for (int i = 0; i < n; ++i) quad.aff.coeffs[i] = grad[i] - hx[i];
    for (int i = 0; i < n; ++i) {
      quad.v1.push_back(vars_[i]);
      quad.v2.push_back(vars_[i]);
      quad.coeffs.push_back(Hp[i][i] / 2);
      for (int j = i + 1; j < n; ++j) {
        quad.v1.push_back(vars_[i]);
        quad.v2.push_back(vars_[j]);
        quad.coeffs.push_back(Hp[i][j]);
      }
    }
  }
  return out;
}

double CostFromErrFunc::value(const Vec& xall) {
  Vec err = f_(gather(xall, vars_));
  double s = 0;
  for (size_t i = 0; i < err.size(); ++i) {
    double e = err[i];
    e = pen_ == SQUARED ? e * e : (pen_ == ABS ? std::fabs(e) : std::max(e, 0.0));
    if (!coeffs_.empty()) e *= coeffs_[i];
    s += e;
  }
  return s;
}
std::shared_ptr<ConvexObjective> CostFromErrFunc::convex(const Vec& xall, Model* model) {
  const Vec x = gather(xall, vars_);
  const std::vector<Vec> jac = dfdx_ ? dfdx_(x) : calcForwardNumJac(f_, x, epsilon_);
  auto out = std::make_shared<ConvexObjective>(model);
  const Vec y = f_(x);
  for (size_t i = 0; i < jac.size(); ++i) {
    AffExpr aff = affFromValGrad(y[i], x, jac[i], vars_);
    double weight = 1;
    if (!coeffs_.empty()) {
      if (coeffs_[i] == 0) continue;
      weight = coeffs_[i];
    }
    if (pen_ == SQUARED) {
      QuadExpr q = exprSquare(aff);
      exprScale(q, weight);
      out->addQuadExpr(q);
    } else if (pen_ == ABS) {
      exprScale(aff, weight);
      out->addAbs(aff, 1);
    } else {
      exprScale(aff, weight);
      out->addHinge(aff, 1);
    }
  }
  return out;
}
Vec ConstraintFromErrFunc::value(const Vec& xall) {
  Vec err = f_(gather(xall, vars_));
  if (!coeffs_.empty())
    for (size_t i = 0; i < err.size(); ++i) err[i] *= coeffs_[i];
  return err;
}
std::shared_ptr<ConvexConstraints> ConstraintFromErrFunc::convex(const Vec& xall, Model*) {
  const Vec x = gather(xall, vars_);
  const std::vector<Vec> jac = dfdx_ ? dfdx_(x) : calcForwardNumJac(f_, x, epsilon_);
  auto out = std::make_shared<ConvexConstraints>();
  const Vec y = f_(x);
  for (size_t i = 0; i < jac.size(); ++i) {
    AffExpr aff = affFromValGrad(y[i], x, jac[i], vars_);
    if (!coeffs_.empty()) {
      if (coeffs_[i] == 0) continue;
      exprScale(aff, coeffs_[i]);
    }
    if (type_ == INEQ)
      out->ineqs.push_back(aff);
    else
      out->eqs.push_back(aff);
  }
  return out;
}

// ============================================================================ SQP driver
// The box of one variable: centred on the iterate clamped into [lb, ub], cut at the variable's own bounds
// (optimizers.cpp:163-168; the identities of trajopt_sqp/test/trust_box_floor_unit.cpp:62-141 hold for it).
void trustBox(double x, double lb, double ub, double trust, double& lo, double& hi) {
  const double xi = std::min(std::max(x, lb), ub);
  lo = std::max(xi - trust, lb);
  hi = std::min(xi + trust, ub);
}
void setTrustBoxConstraints(OptProb& prob, const Vec& x, double trust) {
  const Vec& lb = prob.lower();
  const Vec& ub = prob.upper();
  for (size_t i = 0; i < x.size(); ++i) {
    double lo, hi;
    trustBox(x[i], lb[i], ub[i], trust, lo, hi);
    prob.model()->setVarBounds(static_cast<int>(i), lo, hi);
  }
}

ConvexModels convexifyProblem(OptProb& prob, const Vec& x, const double* merit_coeffs) {
  Model* model = prob.model();
  ConvexModels out;
  model->truncateToPermanent();
  std::vector<std::shared_ptr<ConvexObjective>> cnt_cost_models;
  for (auto& c : prob.getCosts()) out.costs.push_back(c->convex(x, model));
  for (auto& c : prob.getConstraints()) out.cnts.push_back(c->convex(x, model));
  for (size_t c = 0; c < out.cnts.size(); ++c) {
    auto obj = std::make_shared<ConvexObjective>(model);
    for (const AffExpr& a : out.cnts[c]->eqs) obj->addAbs(a, merit_coeffs[c]);
    for (const AffExpr& a : out.cnts[c]->ineqs) obj->addHinge(a, merit_coeffs[c]);
    cnt_cost_models.push_back(obj);
  }
  for (auto& c : out.costs) c->addConstraintsToModel();
  for (auto& c : cnt_cost_models) c->addConstraintsToModel();
  QuadExpr objective;
  for (auto& c : out.costs) exprInc(objective, c->quad);
  for (auto& c : cnt_cost_models) exprInc(objective, c->quad);
  model->setObjective(objective);
  return out;
}
void ConvexModels::values(const double* x, Vec& cost_vals, Vec& cnt_viols) const {
  cost_vals.resize(costs.size());
  cnt_viols.resize(cnts.size());
  for (size_t i = 0; i < costs.size(); ++i) cost_vals[i] = costs[i]->value(x);
  for (size_t i = 0; i < cnts.size(); ++i) cnt_viols[i] = cnts[i]->violation(x);
}

static double vecSum(const Vec& v) {
  double s = 0;
  for (double e : v) s += e;
  return s;
}
static double vecDot(const Vec& a, const Vec& b) {
  double s = 0;
  for (size_t i = 0; i < a.size(); ++i) s += a[i] * b[i];
  return s;
}
static double vecMax(const Vec& v) { return *std::max_element(v.begin(), v.end()); }

OptStatus BasicTrustRegionSQP::optimize() {
  Model* model = prob_->model();
  const auto constraints = prob_->getConstraints();
  const auto& costs = prob_->getCosts();
  Vec merit_error_coeffs(constraints.size(), param_.initial_merit_error_coeff);
  if (results_.x.empty()) throw std::runtime_error("you forgot to initialize!");

  results_.x = prob_->getClosestFeasiblePoint(results_.x);
  OptStatus retval = OPT_INVALID;
  trace.clear();
  records.clear();
  ended = false;
  const auto start = stop_ == STOP_WALL_CLOCK ? std::chrono::steady_clock::now() : std::chrono::steady_clock::time_point();
  const double nan = std::numeric_limits<double>::quiet_NaN();

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
  auto feasible = [&] { return results_.cnt_viols.empty() || vecMax(results_.cnt_viols) < param_.cnt_tolerance; };
  auto failedRecord = [&] {
    return IterRecord{merit_error_coeffs, Vec(costs.size(), nan), Vec(constraints.size(), nan),
                      Vec(costs.size(), nan), Vec(constraints.size(), nan), Vec(results_.x.size(), nan)};
  };

  for (int merit_increases = 0; merit_increases < param_.max_merit_coeff_increases; ++merit_increases) {
    for (int iter = 1;; ++iter) {
      if (results_.cost_vals.empty() && results_.cnt_viols.empty()) {  // first iteration only
        results_.cnt_viols = evalViols(results_.x);
        results_.cost_vals = evalCosts(results_.x);
        ++results_.n_func_evals;
        if (record)
          records.push_back({merit_error_coeffs, Vec(costs.size(), nan), Vec(constraints.size(), nan),
                             results_.cost_vals, results_.cnt_viols, results_.x});
      }
      if (stop_ != STOP_NONE) {  // the iteration top: the stop rule, never on a retry below
        const bool over = stop_ == STOP_QP_BUDGET
                              ? results_.n_qp_solves >= qp_budget_
                              : std::chrono::duration<double>(std::chrono::steady_clock::now() - start).count() > max_time_;
        if (over) {
          ended = true;
          retval = feasible() ? OPT_CONVERGED : OPT_TIME_LIMIT;
          goto cleanup;
        }
      }
      const ConvexModels cm = convexifyProblem(*prob_, results_.x, merit_error_coeffs.data());

      int qp_solver_failures = 0;
      while (param_.trust_box_size >= param_.min_trust_box_size) {
        setTrustBoxConstraints(*prob_, results_.x, param_.trust_box_size);
        const CvxStatus status = model->optimize();
        ++results_.n_qp_solves;
        if (status != CVX_SOLVED) {
          trace.push_back({merit_increases, iter, param_.trust_box_size, 0, 0, 0, model->lastResult().status,
                           model->lastResult().iters, 3});
          if (record) records.push_back(failedRecord());
          if (qp_solver_failures < (param_.max_qp_solver_failures - 1)) {
            param_.trust_box_size *= param_.trust_shrink_ratio;
            qp_solver_failures++;
            continue;
          }
          if (qp_solver_failures == (param_.max_qp_solver_failures - 1)) {
            param_.trust_box_size = param_.min_trust_box_size;
            qp_solver_failures++;
            continue;
          }
          retval = OPT_FAILED;
          goto cleanup;
        }
        // BasicTrustRegionSQPResults::update, optimizers.cpp:380-426
        const Vec& mv = model->solution();
        Vec model_cost_vals, model_cnt_viols;
        cm.values(mv.data(), model_cost_vals, model_cnt_viols);
        Vec new_x(mv.begin(), mv.begin() + static_cast<long>(results_.x.size()));
        const Vec new_cost_vals = evalCosts(new_x);
        const Vec new_cnt_viols = evalViols(new_x);
        const double old_merit = vecSum(results_.cost_vals) + vecDot(results_.cnt_viols, merit_error_coeffs);
        const double model_merit = vecSum(model_cost_vals) + vecDot(model_cnt_viols, merit_error_coeffs);
        const double new_merit = vecSum(new_cost_vals) + vecDot(new_cnt_viols, merit_error_coeffs);
        const double approx_merit_improve = old_merit - model_merit;
        const double exact_merit_improve = old_merit - new_merit;
        const double merit_improve_ratio = exact_merit_improve / approx_merit_improve;
        ++results_.n_func_evals;
        TraceEntry te{merit_increases, iter, param_.trust_box_size, old_merit, model_merit, new_merit,
                      model->lastResult().status, model->lastResult().iters, 0};
        te.pri = model->lastResult().admm_pri;
        te.dua = model->lastResult().admm_dua;
        te.rho = model->lastResult().rho;
        te.polish = model->lastResult().polish;
        te.warm = model->lastResult().warm;
        if (record)
          records.push_back({merit_error_coeffs, model_cost_vals, model_cnt_viols, new_cost_vals, new_cnt_viols, new_x});

        if (approx_merit_improve < param_.min_approx_improve) {
          te.action = 2;
          trace.push_back(te);
          retval = OPT_CONVERGED;
          goto penaltyadjustment;
        }
        if (approx_merit_improve / old_merit < param_.min_approx_improve_frac) {
          te.action = 2;
          trace.push_back(te);
          retval = OPT_CONVERGED;
          goto penaltyadjustment;
        } else if (exact_merit_improve < 0 || merit_improve_ratio < param_.improve_ratio_threshold) {
          param_.trust_box_size *= param_.trust_shrink_ratio;
          te.action = 0;
          trace.push_back(te);
        } else {
          results_.x = new_x;
          results_.cost_vals = new_cost_vals;
          results_.cnt_viols = new_cnt_viols;
          param_.trust_box_size *= param_.trust_expand_ratio;
          te.action = 1;
          trace.push_back(te);
          break;
        }
      }
      if (param_.trust_box_size < param_.min_trust_box_size) {
        retval = OPT_CONVERGED;
        goto penaltyadjustment;
      } else if (iter >= param_.max_iter) {
        retval = OPT_SCO_ITERATION_LIMIT;
        if (feasible()) retval = OPT_CONVERGED;
        goto cleanup;
      }
    }
  penaltyadjustment:
    if (feasible()) {
      goto cleanup;
    } else {
      if (param_.inflate_constraints_individually) {
        for (size_t i = 0; i < results_.cnt_viols.size(); ++i)
          if (results_.cnt_viols[i] > param_.cnt_tolerance) merit_error_coeffs[i] *= param_.merit_coeff_increase_ratio;
      } else {
        for (double& c : merit_error_coeffs) c *= param_.merit_coeff_increase_ratio;
      }
      param_.trust_box_size =
          std::fmax(param_.trust_box_size, param_.min_trust_box_size / param_.trust_shrink_ratio * 1.5);
    }
  }
  retval = OPT_PENALTY_ITERATION_LIMIT;
cleanup:
  results_.status = retval;
  results_.total_cost = vecSum(results_.cost_vals);
  return retval;
}

}  // namespace oracle
