// General (dense) QP entry point behind the sco::Model plugin surface (include/trajopt_b200_sco.hpp):
//   min 1/2 x'Px + q'x   s.t.  l <= Ax <= u        (OSQP's canonical form, osqp_interface.cpp:170-281: the variable bounds
//                                                   are identity rows of A)
// solved by the same OSQP-equivalent ADMM as the trajectory QPs (Ruiz equilibration, rho_eq = 1e3 rho on equality rows,
// alpha = 1.6, termination + infeasibility certificates every check_termination iterations, adaptive rho, polish with KKT
// verification and ADMM continuation — DESIGN.md section 6), restated for an arbitrary dense P and A: one CTA per QP,
// the reduced KKT matrix  K = P + sigma I + A' diag(rho) A  factored by a dense Cholesky (K is SPD) so that an ADMM
// iteration is dense products and two triangular solves.  This is the compatibility surface (a sco::Model::optimize() call at a time, what
// trajopt_sco's own SQP loop issues); the batched trajectory path does not go through it.
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "../../include/trajopt_b200.h"

namespace {
constexpr int kThreads = 256;
constexpr double kInf = 1e30, kMinScaling = 1e-4, kMaxScaling = 1e4;
constexpr double kRhoMin = 1e-6, kRhoMax = 1e6, kRhoTol = 1e-4, kRhoEq = 1e3, kVerifyTol = 1e-9;
constexpr int kVerifyRounds = 3;
constexpr long long kMaxDenseEntries = 2147483647LL;
enum { S_UNSOLVED = 0, S_SOLVED = 1, S_SOLVED_INACC = 2, S_PINF = 3, S_PINF_INACC = 4, S_DINF = 5, S_DINF_INACC = 6, S_MAXITER = 7, S_NONCVX = 8 };

struct GqDev {
  int n, m, batch;
  const double *P, *q, *A, *l, *u;  // [batch] problems back to back
  double* ws;                       // workspace, ws_stride doubles per problem
  size_t ws_stride;
  tb200_qp_settings st;
  double *x_out, *y_out;
  int *status_out, *iters_out, *polish_out;
};

__device__ __forceinline__ double limit_scaling(double v) {
  v = v < kMinScaling ? 1.0 : v;
  return v > kMaxScaling ? kMaxScaling : v;
}

struct Red {
  double* buf;  // shared [kThreads / 32]
  int tid;
  // block-wide max / sum (every thread gets the result); fixed order
  __device__ double run(double v, bool sum) const {
    for (int o = 16; o > 0; o >>= 1) {
      const double w = __shfl_xor_sync(0xffffffffu, v, o);
      v = sum ? v + w : fmax(v, w);
    }
    __syncthreads();
    if ((tid & 31) == 0) buf[tid >> 5] = v;
    __syncthreads();
    double a = buf[0];
    for (int w = 1; w < kThreads / 32; ++w) a = sum ? a + buf[w] : fmax(a, buf[w]);
    return a;
  }
  __device__ double max(double v) const { return run(v, false); }
  __device__ double sum(double v) const { return run(v, true); }
};

__global__ void __launch_bounds__(kThreads, 1) general_qp_kernel(const __grid_constant__ GqDev g) {
  __shared__ double s_red[kThreads / 32];
  __shared__ unsigned long long s_h[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, b = blockIdx.x;
  const int n = g.n, m = g.m;
  const tb200_qp_settings& st = g.st;
  const Red red{s_red, tid};
  // ---- workspace carve-up ------------------------------------------------------------------------------------------
  double* w = g.ws + static_cast<size_t>(b) * g.ws_stride;
  auto take = [&](size_t cnt) {
    double* p = w;
    w += (cnt + 1) & ~static_cast<size_t>(1);
    return p;
  };
  double* Ps = take(static_cast<size_t>(n) * n);  // scaled P (full symmetric)
  double* As = take(static_cast<size_t>(m) * n);  // scaled A (row major)
  double* K = take(static_cast<size_t>(n) * n);   // Cholesky factor of the current reduced KKT matrix (L and L')
  double *qs = take(n), *D = take(n), *x = take(n), *xt = take(n), *rhs = take(n), *tmpn = take(n), *Px = take(n), *Aty = take(n),
         *dx = take(n), *xq = take(n), *rd = take(n), *stepv = take(n), *colk = take(n), *sx = take(n);
  double *ls = take(m), *us = take(m), *E = take(m), *rho_vec = take(m), *z = take(m), *y = take(m), *zt = take(m), *tmpm = take(m),
         *Ax = take(m), *dy = take(m), *wact = take(m), *bb = take(m), *act = take(m), *yq = take(m), *sz = take(m), *sy = take(m);
  const double* P0 = g.P + static_cast<size_t>(b) * n * n;
  const double* A0 = g.A + static_cast<size_t>(b) * m * n;

  // ---- dense products (coalesced: consecutive threads read consecutive columns) --------------------------------------
  auto sym_mv = [&](const double* M, const double* in, double* out) {  // out = M in, M symmetric: column walk = row walk
    for (int i = tid; i < n; i += kThreads) {
      double s = 0.0;
      for (int j = 0; j < n; ++j) s += M[static_cast<size_t>(j) * n + i] * in[j];
      out[i] = s;
    }
    __syncthreads();
  };
  auto At_mv = [&](const double* in, double* out) {  // out[n] = As' in[m]
    for (int j = tid; j < n; j += kThreads) {
      double s = 0.0;
      for (int r = 0; r < m; ++r) s += As[static_cast<size_t>(r) * n + j] * in[r];
      out[j] = s;
    }
    __syncthreads();
  };
  auto A_mv = [&](const double* in, double* out) {  // out[m] = As in[n]: one warp per row, lanes over the columns
    for (int r = wid; r < m; r += kThreads / 32) {
      double s = 0.0;
      for (int j = lane; j < n; j += 32) s += As[static_cast<size_t>(r) * n + j] * in[j];
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) out[r] = s;
    }
    __syncthreads();
  };
  // K <- Cholesky factor of Ps + sig I + As' diag(wts) As, L in the lower triangle and L' in the upper (so that both
  // triangular solves walk rows: coalesced); false when the matrix is not positive definite.  A factor, not an explicit
  // inverse: the ADMM matrix (rho_eq = 1e3 rho up to 1e6) and the polish matrix (1/delta = 1e6 on the active rows) reach
  // condition numbers of 1e12 and more on penalty QPs whose P is singular on the slacks, where an explicit inverse loses
  // every digit and the Cholesky solve stays backward stable.
  auto assemble_factor = [&](double sig, const double* wts) -> bool {
    for (int e = tid; e < n * n; e += kThreads) {
      const int i = e / n, j = e % n;
      double s = Ps[e] + (i == j ? sig : 0.0);
      for (int r = 0; r < m; ++r) {
        const double wr = wts[r];
        if (wr != 0.0) s += As[static_cast<size_t>(r) * n + i] * wr * As[static_cast<size_t>(r) * n + j];
      }
      K[e] = s;
    }
    __syncthreads();
    for (int k = 0; k < n; ++k) {  // right-looking, on the upper triangle: row k of U = L' is column k of L
      const double piv = K[static_cast<size_t>(k) * n + k];
      __syncthreads();            // every thread has read the pivot before row k is overwritten
      if (!(piv > 0.0)) return false;  // every thread read the same pivot: a uniform exit
      const double lkk = sqrt(piv), il = 1.0 / lkk;
      for (int j = k + tid; j < n; j += kThreads) K[static_cast<size_t>(k) * n + j] = j == k ? lkk : K[static_cast<size_t>(k) * n + j] * il;
      __syncthreads();
      const int r = n - k - 1;
      for (int e = tid; e < r * r; e += kThreads) {
        const int i = k + 1 + e / r, j = k + 1 + e % r;
        if (j >= i) K[static_cast<size_t>(i) * n + j] -= K[static_cast<size_t>(k) * n + i] * K[static_cast<size_t>(k) * n + j];
      }
      __syncthreads();
    }
    for (int e = tid; e < n * n; e += kThreads) {  // mirror: K[i][j] = L[i][j] below the diagonal
      const int i = e / n, j = e % n;
      if (i > j) K[e] = K[static_cast<size_t>(j) * n + i];
    }
    __syncthreads();
    return true;
  };
  // out = (L L')^-1 in with the factor of assemble_factor; in and out distinct, colk is scratch
  auto chol_solve = [&](const double* in, double* out) {
    for (int i = tid; i < n; i += kThreads) colk[i] = in[i];
    __syncthreads();
    for (int k = 0; k < n; ++k) {  // L w = in: colk[k] is final once step k - 1 is done
      const double wk = colk[k] / K[static_cast<size_t>(k) * n + k];
      for (int i = k + 1 + tid; i < n; i += kThreads) colk[i] -= K[static_cast<size_t>(k) * n + i] * wk;
      if (tid == 0) out[k] = wk;
      __syncthreads();
    }
    for (int i = tid; i < n; i += kThreads) colk[i] = out[i];
    __syncthreads();
    for (int k = n - 1; k >= 0; --k) {  // L' x = w: row k of L holds column k of L'
      const double xk = colk[k] / K[static_cast<size_t>(k) * n + k];
      for (int i = tid; i < k; i += kThreads) colk[i] -= K[static_cast<size_t>(k) * n + i] * xk;
      if (tid == 0) out[k] = xk;
      __syncthreads();
    }
  };

  // ---- copy + Ruiz equilibration (scale_data of OSQP; same passes as the trajectory kernel's qp_scale) --------------
  for (int e = tid; e < n * n; e += kThreads) {
    const int i = e / n, j = e % n;
    Ps[e] = (j >= i) ? P0[e] : P0[static_cast<size_t>(j) * n + i];  // the upper triangle is the data
  }
  for (int e = tid; e < m * n; e += kThreads) As[e] = A0[e];
  for (int i = tid; i < n; i += kThreads) {
    qs[i] = g.q[static_cast<size_t>(b) * n + i];
    D[i] = 1.0;
  }
  for (int r = tid; r < m; r += kThreads) {
    ls[r] = fmax(g.l[static_cast<size_t>(b) * m + r], -kInf);
    us[r] = fmin(g.u[static_cast<size_t>(b) * m + r], kInf);
    E[r] = 1.0;
  }
  double c = 1.0;
  __syncthreads();
  for (int pass = 0; pass < st.scaling; ++pass) {
    for (int j = tid; j < n; j += kThreads) {  // column norms of [P A'; A 0]
      double v = 0.0;
      for (int i = 0; i < n; ++i) v = fmax(v, fabs(Ps[static_cast<size_t>(i) * n + j]));
      for (int r = 0; r < m; ++r) v = fmax(v, fabs(As[static_cast<size_t>(r) * n + j]));
      tmpn[j] = 1.0 / sqrt(limit_scaling(v));
    }
    for (int r = wid; r < m; r += kThreads / 32) {
      double v = 0.0;
      for (int j = lane; j < n; j += 32) v = fmax(v, fabs(As[static_cast<size_t>(r) * n + j]));
      for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
      if (lane == 0) tmpm[r] = 1.0 / sqrt(limit_scaling(v));
    }
    __syncthreads();
    for (int e = tid; e < n * n; e += kThreads) Ps[e] *= tmpn[e / n] * tmpn[e % n];
    for (int e = tid; e < m * n; e += kThreads) As[e] *= tmpm[e / n] * tmpn[e % n];
    for (int i = tid; i < n; i += kThreads) {
      qs[i] *= tmpn[i];
      D[i] *= tmpn[i];
    }
    for (int r = tid; r < m; r += kThreads) E[r] *= tmpm[r];
    __syncthreads();
    double cs = 0.0, qn = 0.0;  // cost normalisation: mean column inf-norm of P against the inf-norm of q
    for (int j = tid; j < n; j += kThreads) {
      double v = 0.0;
      for (int i = 0; i < n; ++i) v = fmax(v, fabs(Ps[static_cast<size_t>(i) * n + j]));
      cs += v;
      qn = fmax(qn, fabs(qs[j]));
    }
    const double mean = limit_scaling(red.sum(cs) / n);
    const double ct = 1.0 / fmax(mean, limit_scaling(red.max(qn)));
    for (int e = tid; e < n * n; e += kThreads) Ps[e] *= ct;
    for (int i = tid; i < n; i += kThreads) qs[i] *= ct;
    c *= ct;
    __syncthreads();
  }
  const double cinv = 1.0 / c;
  for (int r = tid; r < m; r += kThreads) {
    ls[r] *= E[r];
    us[r] *= E[r];
  }
  __syncthreads();

  // ---- rho vector (equality rows 1e3 rho, free rows rho_min) ---------------------------------------------------------
  double rho = fmin(fmax(st.rho, kRhoMin), kRhoMax);
  auto set_rho = [&]() {
    for (int r = tid; r < m; r += kThreads) {
      const bool free_row = ls[r] < -kInf * kMinScaling && us[r] > kInf * kMinScaling;
      rho_vec[r] = free_row ? kRhoMin : ((us[r] - ls[r] < kRhoTol) ? kRhoEq * rho : rho);
    }
    __syncthreads();
  };
  set_rho();
  for (int i = tid; i < n; i += kThreads) x[i] = 0.0;
  for (int r = tid; r < m; r += kThreads) z[r] = y[r] = 0.0;
  __syncthreads();

  int status = S_UNSOLVED, iter = 0, polish = 0, round = 0;
  double pri_res = 0.0, dua_res = 0.0, eps_scale = 1.0, pp = 0.0, pdres = 0.0;
  bool early_verified = false;
  unsigned long long prev_guess = 0ull, failed_guess = 0ull, pending_guess = 0ull;
  bool have_prev = false, have_failed = false;
  if (!assemble_factor(st.sigma, rho_vec)) status = S_NONCVX;

  auto update_info = [&]() {
    A_mv(x, Ax);
    sym_mv(Ps, x, Px);
    At_mv(y, Aty);
    double p = 0.0, d = 0.0;
    for (int r = tid; r < m; r += kThreads) p = fmax(p, fabs((Ax[r] - z[r]) / E[r]));
    for (int i = tid; i < n; i += kThreads) d = fmax(d, fabs((qs[i] + Px[i] + Aty[i]) / D[i]));
    pri_res = red.max(p);
    dua_res = red.max(d) * cinv;
  };
  auto primal_infeasible = [&](double eps) -> bool {
    double nd = 0.0, lhs = 0.0;
    for (int r = tid; r < m; r += kThreads) {
      double d = dy[r];
      if (us[r] > kInf * kMinScaling) d = (ls[r] < -kInf * kMinScaling) ? 0.0 : fmin(d, 0.0);
      else if (ls[r] < -kInf * kMinScaling) d = fmax(d, 0.0);
      tmpm[r] = d;
      nd = fmax(nd, fabs(E[r] * d));
      lhs += us[r] * fmax(d, 0.0) + ls[r] * fmin(d, 0.0);
    }
    nd = red.max(nd);
    lhs = red.sum(lhs);
    if (!(nd > eps && lhs < -eps * nd)) return false;
    __syncthreads();
    At_mv(tmpm, tmpn);
    double a = 0.0;
    for (int i = tid; i < n; i += kThreads) a = fmax(a, fabs(tmpn[i] / D[i]));
    return red.max(a) < eps * nd;
  };
  auto dual_infeasible = [&](double eps) -> bool {
    double ndx = 0.0, qdx = 0.0;
    for (int i = tid; i < n; i += kThreads) {
      ndx = fmax(ndx, fabs(D[i] * dx[i]));
      qdx += qs[i] * dx[i];
    }
    ndx = red.max(ndx);
    qdx = red.sum(qdx);
    if (!(ndx > eps && qdx < -c * eps * ndx)) return false;
    sym_mv(Ps, dx, tmpn);
    double a = 0.0;
    for (int i = tid; i < n; i += kThreads) a = fmax(a, fabs(tmpn[i] / D[i]));
    if (!(red.max(a) < c * eps * ndx)) return false;
    A_mv(dx, tmpm);
    double bad = 0.0;
    for (int r = tid; r < m; r += kThreads) {
      const double v = tmpm[r] / E[r];
      if ((us[r] < kInf * kMinScaling && v > eps * ndx) || (ls[r] > -kInf * kMinScaling && v < -eps * ndx)) bad += 1.0;
    }
    return red.sum(bad) == 0.0;
  };
  auto check_termination = [&](bool approximate) -> int {
    double eps_abs = st.eps_abs * eps_scale, eps_rel = st.eps_rel * eps_scale, epi = st.eps_prim_inf, edi = st.eps_dual_inf;
    if (approximate) {
      eps_abs *= 10; eps_rel *= 10; epi *= 10; edi *= 10;
    }
    if (pri_res > kInf || dua_res > kInf) return S_NONCVX;
    double nz = 0.0, nax = 0.0, nq = 0.0, naty = 0.0, npx = 0.0;
    for (int r = tid; r < m; r += kThreads) {
      nz = fmax(nz, fabs(z[r] / E[r]));
      nax = fmax(nax, fabs(Ax[r] / E[r]));
    }
    for (int i = tid; i < n; i += kThreads) {
      nq = fmax(nq, fabs(qs[i] / D[i]));
      naty = fmax(naty, fabs(Aty[i] / D[i]));
      npx = fmax(npx, fabs(Px[i] / D[i]));
    }
    nz = red.max(nz); nax = red.max(nax); nq = red.max(nq); naty = red.max(naty); npx = red.max(npx);
    const double eps_pri = eps_abs + eps_rel * fmax(nz, nax);
    const double eps_dua = eps_abs + eps_rel * cinv * fmax(nq, fmax(naty, npx));
    const bool pri_ok = pri_res < eps_pri, dua_ok = dua_res < eps_dua;
    bool pinf = false, dinf = false;
    if (!pri_ok) pinf = primal_infeasible(epi);
    if (!dua_ok) dinf = dual_infeasible(edi);
    if (pri_ok && dua_ok) return approximate ? S_SOLVED_INACC : S_SOLVED;
    if (pinf) return approximate ? S_PINF_INACC : S_PINF;
    if (dinf) return approximate ? S_DINF_INACC : S_DINF;
    return S_UNSOLVED;
  };
  auto guess_hash = [&]() -> unsigned long long {  // order-independent hash of the active-set guess (optimisation O1)
    unsigned long long h = 0ull;
    for (int r = tid; r < m; r += kThreads) {
      int a = 0;
      if (z[r] - ls[r] < -y[r]) a = -1;
      else if (us[r] - z[r] < y[r]) a = 1;
      if (a) {
        unsigned long long v = 2ull * r + (a > 0 ? 1ull : 0ull) + 0x9e3779b97f4a7c15ull;
        v = (v ^ (v >> 30)) * 0xbf58476d1ce4e5b9ull;
        v = (v ^ (v >> 27)) * 0x94d049bb133111ebull;
        h += v ^ (v >> 31);
      }
    }
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    __syncthreads();
    if (lane == 0) s_h[wid] = h;
    __syncthreads();
    h = 0ull;
    for (int k = 0; k < kThreads / 32; ++k) h += s_h[k];
    return h;
  };
  // polish (OSQP polish.c): equality-constrained QP on the guessed active set in reduced form, iterative refinement,
  // KKT verification of the result (deviation D2); the ADMM iterate is untouched (the polish works on xq, yq)
  auto polish_once = [&](bool& verified) -> bool {
    verified = false;
    for (int r = tid; r < m; r += kThreads) {
      int a = 0;
      if (z[r] - ls[r] < -y[r]) a = -1;
      else if (us[r] - z[r] < y[r]) a = 1;
      wact[r] = a ? 1.0 / st.delta : 0.0;
      bb[r] = a < 0 ? ls[r] : us[r];
      act[r] = a;
      yq[r] = 0.0;
    }
    for (int i = tid; i < n; i += kThreads) xq[i] = 0.0;
    __syncthreads();
    if (!assemble_factor(st.delta, wact)) return false;
    for (int it = 0; it <= st.polish_refine_iter; ++it) {
      sym_mv(Ps, xq, Px);
      At_mv(yq, Aty);
      A_mv(xq, Ax);
      for (int r = tid; r < m; r += kThreads) tmpm[r] = wact[r] * (Ax[r] - bb[r]);
      __syncthreads();
      At_mv(tmpm, tmpn);
      for (int i = tid; i < n; i += kThreads) rd[i] = -(Px[i] + qs[i] + Aty[i]) - tmpn[i];
      __syncthreads();
      chol_solve(rd, stepv);
      for (int i = tid; i < n; i += kThreads) xq[i] += stepv[i];
      __syncthreads();
      A_mv(xq, Ax);
      for (int r = tid; r < m; r += kThreads)
        if (wact[r] != 0.0) yq[r] += wact[r] * (Ax[r] - bb[r]);
      __syncthreads();
    }
    A_mv(xq, Ax);
    sym_mv(Ps, xq, Px);
    At_mv(yq, Aty);
    double p = 0.0, d = 0.0, bad = 0.0;
    for (int r = tid; r < m; r += kThreads) {
      const double zr = fmin(fmax(Ax[r], ls[r]), us[r]);
      p = fmax(p, fabs((Ax[r] - zr) / E[r]));
      if (act[r] != 0.0 && us[r] - ls[r] >= kRhoTol) {
        if (act[r] > 0 && yq[r] < -kVerifyTol) bad += 1.0;
        if (act[r] < 0 && yq[r] > kVerifyTol) bad += 1.0;
      }
    }
    for (int i = tid; i < n; i += kThreads) d = fmax(d, fabs((qs[i] + Px[i] + Aty[i]) / D[i]));
    pp = red.max(p);
    pdres = red.max(d) * cinv;
    bad = red.sum(bad);
    verified = bad == 0.0 && pp <= kVerifyTol && isfinite(pp) && isfinite(pdres);
    return true;
  };

  // ---- main loop: ADMM -> polish -> verify; on a failed verification ADMM continues with 10x tighter tolerances ------
  bool done = status != S_UNSOLVED;
  while (!done) {
    status = S_UNSOLVED;
    bool stop = false;
    while (!stop) {
      if (iter >= st.max_iter) {
        if (!(st.check_termination > 0 && iter % st.check_termination == 0)) update_info();
        status = check_termination(true);
        if (status == S_UNSOLVED) status = S_MAXITER;
        break;
      }
      ++iter;
      // update_xz_tilde: K xt = sigma x - q + A'(rho z - y); zt = A xt; relaxation, projection, dual update
      for (int r = tid; r < m; r += kThreads) tmpm[r] = rho_vec[r] * z[r] - y[r];
      __syncthreads();
      At_mv(tmpm, rhs);
      for (int i = tid; i < n; i += kThreads) rhs[i] += st.sigma * x[i] - qs[i];
      __syncthreads();
      chol_solve(rhs, xt);
      A_mv(xt, zt);
      for (int i = tid; i < n; i += kThreads) {
        const double xn = st.alpha * xt[i] + (1.0 - st.alpha) * x[i];
        dx[i] = xn - x[i];
        x[i] = xn;
      }
      for (int r = tid; r < m; r += kThreads) {
        const double zr = st.alpha * zt[r] + (1.0 - st.alpha) * z[r];
        double v = zr + y[r] / rho_vec[r];
        v = fmin(fmax(v, ls[r]), us[r]);
        z[r] = v;
        dy[r] = rho_vec[r] * (zr - v);
        y[r] += dy[r];
      }
      __syncthreads();
      const bool can_check = st.check_termination > 0 && iter % st.check_termination == 0;
      if (can_check) {
        update_info();
        status = check_termination(false);
        if (status != S_UNSOLVED) break;
        bool try_early = st.polishing && st.early_polish_every > 0 && iter >= st.early_polish_from && iter % st.early_polish_every == 0;
        if (try_early) {
          const unsigned long long h = guess_hash();
          const bool stable = have_prev && h == prev_guess;
          prev_guess = h;
          have_prev = true;
          try_early = stable && !(have_failed && h == failed_guess);
          pending_guess = h;
        }
        if (try_early) {
          bool verified = false;
          const bool factored = polish_once(verified);
          if (factored && verified) {
            early_verified = true;
            status = S_SOLVED;
            break;
          }
          failed_guess = pending_guess;
          have_failed = true;
          update_info();
          if (!assemble_factor(st.sigma, rho_vec)) {
            status = S_NONCVX;
            break;
          }
        }
      }
      if (st.adaptive_rho && st.adaptive_rho_interval > 0 && iter % st.adaptive_rho_interval == 0) {
        if (!can_check) update_info();
        double p = 0.0, d = 0.0, nz = 0.0, nax = 0.0, nq = 0.0, naty = 0.0, npx = 0.0;
        for (int r = tid; r < m; r += kThreads) {
          p = fmax(p, fabs(Ax[r] - z[r]));
          nz = fmax(nz, fabs(z[r]));
          nax = fmax(nax, fabs(Ax[r]));
        }
        for (int i = tid; i < n; i += kThreads) {
          d = fmax(d, fabs(qs[i] + Px[i] + Aty[i]));
          nq = fmax(nq, fabs(qs[i]));
          naty = fmax(naty, fabs(Aty[i]));
          npx = fmax(npx, fabs(Px[i]));
        }
        p = red.max(p); d = red.max(d); nz = red.max(nz); nax = red.max(nax); nq = red.max(nq); naty = red.max(naty); npx = red.max(npx);
        p /= (fmax(nz, nax) + 1e-10);
        d /= (fmax(nq, fmax(naty, npx)) + 1e-10);
        double rho_new = rho * sqrt(p / (d + 1e-10));
        rho_new = fmin(fmax(rho_new, kRhoMin), kRhoMax);
        if (rho_new > rho * st.adaptive_rho_tolerance || rho_new < rho / st.adaptive_rho_tolerance) {
          rho = rho_new;
          set_rho();
          if (!assemble_factor(st.sigma, rho_vec)) {
            status = S_NONCVX;
            break;
          }
        }
      }
    }
    if (status != S_SOLVED || !st.polishing) break;
    if (early_verified) {
      polish = 1;
      break;
    }
    bool verified = false;
    const bool factored = polish_once(verified);
    if (factored && verified) {
      polish = 1;
      break;
    }
    if (round >= kVerifyRounds || iter >= st.max_iter) {  // OSQP's own acceptance rule
      const bool ok = factored && ((pp < pri_res && pdres < dua_res) || (pp < pri_res && dua_res < 1e-10) ||
                                   (pdres < dua_res && pri_res < 1e-10)) && isfinite(pp) && isfinite(pdres);
      polish = ok ? 2 : -1;
      break;
    }
    ++round;
    eps_scale *= 0.1;
    if (!assemble_factor(st.sigma, rho_vec)) {
      status = S_NONCVX;
      break;
    }
  }
  (void)sx; (void)sz; (void)sy;
  // ---- unscale and store ---------------------------------------------------------------------------------------------
  const double* xs = polish > 0 ? xq : x;
  const double* ys = polish > 0 ? yq : y;
  for (int i = tid; i < n; i += kThreads) g.x_out[static_cast<size_t>(b) * n + i] = D[i] * xs[i];
  for (int r = tid; r < m; r += kThreads) g.y_out[static_cast<size_t>(b) * m + r] = cinv * E[r] * ys[r];
  if (tid == 0) {
    g.status_out[b] = status;
    g.iters_out[b] = iter;
    g.polish_out[b] = polish;
  }
}

thread_local std::string g_gq_err;
}  // namespace

extern "C" {

const char* tb200_qp_general_last_error(void) { return g_gq_err.c_str(); }

int tb200_qp_solve_general(const tb200_qp_general* qp, const tb200_qp_settings* settings, int device, double* x, double* y,
                           int32_t* status, int32_t* iters, int32_t* polish) {
  auto fail = [](int code, const std::string& msg) {
    g_gq_err = msg;
    return code;
  };
  if (!qp || !x || !status) return fail(TB200_ERR_INVALID, "null argument");
  const int n = qp->n, m = qp->m, B = qp->batch < 1 ? 1 : qp->batch;
  if (n < 1 || m < 0) return fail(TB200_ERR_INVALID, "n must be >= 1 and m >= 0");
  if (!qp->P || !qp->q || (m > 0 && (!qp->A || !qp->l || !qp->u))) return fail(TB200_ERR_INVALID, "null QP data");
  // the kernel indexes P, K and A with 32-bit n * n and m * n (one CTA per QP: far beyond any size it is meant for)
  if (static_cast<long long>(n) * n > kMaxDenseEntries || static_cast<long long>(m) * n > kMaxDenseEntries)
    return fail(TB200_ERR_UNSUPPORTED, "general QP too large: n * n and m * n must each be at most 2^31 - 1");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(TB200_ERR_NO_DEVICE, "no CUDA device: trajopt_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(TB200_ERR_INVALID, "bad device ordinal");
#define GCK(call)                                                                                  \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(TB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)
  GCK(cudaSetDevice(device));
  tb200_qp_settings st;
  if (settings) st = *settings;
  else tb200_default_qp_settings(&st);
  const size_t nn = static_cast<size_t>(n) * n, mn = static_cast<size_t>(m) * n;
  const size_t ws = 2 * (nn + 2) + (mn + 2) + 14 * (static_cast<size_t>(n) + 2) + 16 * (static_cast<size_t>(m) + 2);
  double *dP = nullptr, *dq = nullptr, *dA = nullptr, *dl = nullptr, *du = nullptr, *dws = nullptr, *dx = nullptr, *dy = nullptr;
  int* dint = nullptr;
  auto release = [&]() {
    cudaFree(dP); cudaFree(dq); cudaFree(dA); cudaFree(dl); cudaFree(du); cudaFree(dws); cudaFree(dx); cudaFree(dy); cudaFree(dint);
  };
  cudaError_t e = cudaSuccess;
  auto alloc = [&](double** p, size_t cnt) {
    if (e == cudaSuccess) e = cudaMalloc(p, std::max<size_t>(cnt, 1) * sizeof(double));
  };
  alloc(&dP, B * nn); alloc(&dq, static_cast<size_t>(B) * n); alloc(&dA, B * mn); alloc(&dl, static_cast<size_t>(B) * m);
  alloc(&du, static_cast<size_t>(B) * m); alloc(&dws, B * ws); alloc(&dx, static_cast<size_t>(B) * n); alloc(&dy, static_cast<size_t>(B) * std::max(m, 1));
  if (e == cudaSuccess) e = cudaMalloc(&dint, 3 * static_cast<size_t>(B) * sizeof(int));
  if (e != cudaSuccess) {
    release();
    return fail(TB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  auto up = [&](double* d, const double* h, size_t cnt) {
    if (e == cudaSuccess && cnt) e = cudaMemcpy(d, h, cnt * sizeof(double), cudaMemcpyHostToDevice);
  };
  up(dP, qp->P, B * nn); up(dq, qp->q, static_cast<size_t>(B) * n); up(dA, qp->A, B * mn); up(dl, qp->l, static_cast<size_t>(B) * m);
  up(du, qp->u, static_cast<size_t>(B) * m);
  if (e == cudaSuccess) {
    GqDev g{n, m, B, dP, dq, dA, dl, du, dws, ws, st, dx, dy, dint, dint + B, dint + 2 * B};
    general_qp_kernel<<<B, kThreads>>>(g);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  }
  std::vector<int> hint(3 * static_cast<size_t>(B));
  if (e == cudaSuccess) e = cudaMemcpy(x, dx, static_cast<size_t>(B) * n * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && y && m > 0) e = cudaMemcpy(y, dy, static_cast<size_t>(B) * m * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(hint.data(), dint, hint.size() * sizeof(int), cudaMemcpyDeviceToHost);
  release();
  if (e != cudaSuccess) return fail(TB200_ERR_CUDA, std::string("general QP: ") + cudaGetErrorString(e));
  for (int b = 0; b < B; ++b) {
    status[b] = hint[b];
    if (iters) iters[b] = hint[B + b];
    if (polish) polish[b] = hint[2 * B + b];
  }
  return TB200_OK;
#undef GCK
}

}  // extern "C"
