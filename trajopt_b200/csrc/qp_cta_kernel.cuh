// QP subproblem step (qp_step), latency-optimised: one 256-thread CTA works on one trajectory's QP.  A device
// function: solve_kernel.cuh calls it from its persistent loop (and, with the override arguments, for the kernel-level
// entry point tb200_qp_solve_batch).
//
// Replaces OSQPModel::optimize() -> osqp_setup/osqp_solve (trajopt_sco/src/osqp_interface.cpp:283-615) for
// every trajectory of the batch (same algorithm and arithmetic as the oracle's qp_solve: Ruiz equilibration,
// OSQP-equivalent ADMM, adaptive rho, verified polish; see DESIGN.md §4).
//
// Why a CTA per trajectory.  At batch 1024 the wall time of a batched solve is the slowest trajectory's
// sequential chain of ADMM iterations (~8x the mean) times the latency of one iteration.  So the kernel is
// built for per-trajectory latency: 8 warps work on ONE reduced KKT system,
//   (P + sigma I + A' diag(rho) A) x = rhs,   N = T*D unknowns, block tridiagonal with nb = 2*D blocks,
// which is factored and solved by BLOCK CYCLIC REDUCTION: log2(M) levels instead of M sequential block
// steps (M = N/nb = 15 for 7-DOF x 30).  Level l eliminates every other remaining block p with
//   Ainv_p = A_p^-1,  Um_p = L_p' Ainv_p,  Up_p = L_{p+s} Ainv_p,   (L_p = K(p, p-s), s = 2^l)
//   A_{p-s} -= Um_p L_p,  A_{p+s} -= Up_p L_{p+s}',  L'_{p+s} = -Up_p L_p
// and a solve is  rhs_{p-+s} -= U rhs_p  going down,  x_p = Ainv_p rhs_p - Um_p' x_{p-s} - Up_p' x_{p+s}  going up:
// 2*log2(M)+1 dependent mat-vec steps of 14..42 terms, two threads per (block,row).
//
// Everything an ADMM iteration touches is in shared memory: the factor (3 x M x nb x nb), the trajectory
// vectors, and - when the QP has at most `row_cap` rows, the common case - the rows of the QP themselves.
// The hinge / abs auxiliary variables of the l1 penalty are eliminated per row in closed form (cancellation
// free), exactly as in DESIGN.md §4.2.
//
// Short trajectories (M <= 15 blocks of 14, rows on chip: the headline case) keep their ADMM system in another form,
// the partition inverse (PinvPlan below): a solve is two dependent steps instead of seven; the cyclic reduction stays
// for their polish system and for everything larger.
//
// Sizes.  The level loops of the factorisation and of the generic solve run over task chunks, so the number of
// blocks M is not tied to the CTA size (configs[3]: 50 waypoints = 25 blocks of 14).  Without the partition form the
// register-resident solve of the ADMM loop is used whenever its roles fit the 256 threads (M <= 15 at 7 joints), the
// generic solve (factor rows read from memory) otherwise.  With 14 joints (blocks of 28, configs[4]) the factor (3*M*28*28 doubles = 376 KB at
// 40 waypoints) does not fit shared memory: it lives in a per-CTA region of global memory that stays L2 resident
// (template flag FG), everything else is unchanged.
#pragma once
#include "device_types.cuh"
#include "joint_terms.cuh"

namespace tb200 {

#ifdef TB200_PROFILE
static __device__ unsigned long long g_prof[32];
#define PROF_T0() const long long prof_t0_ = clock64()
#define PROF_ADD(slot) do { if (q.tid == 0) atomicAdd(&g_prof[slot], (unsigned long long)(clock64() - prof_t0_)); } while (0)
#define PROF_COUNT(slot) do { if (q.tid == 0) atomicAdd(&g_prof[slot], 1ull); } while (0)
// the same cycles into two slots (a total and its share of one kind)
#define PROF_ADD2(slot, slot2) do { if (q.tid == 0) { const unsigned long long d_ = clock64() - prof_t0_; \
    atomicAdd(&g_prof[slot], d_); atomicAdd(&g_prof[slot2], d_); } } while (0)
#else
#define PROF_T0()
#define PROF_ADD(slot)
#define PROF_COUNT(slot)
#define PROF_ADD2(slot, slot2)
#endif
// -DTB200_PROFILE_CHECK: the per-level slots of the solve (4, 14, 15, 9) count the parts of a termination check instead
#if defined(TB200_PROFILE) && defined(TB200_PROFILE_CHECK)
#define PROF_CHK_T0() long long pc_ = clock64()
#define PROF_CHK(slot) do { const long long n_ = clock64(); if (q.tid == 0) atomicAdd(&g_prof[slot], (unsigned long long)(n_ - pc_)); pc_ = n_; } while (0)
#else
#define PROF_CHK_T0()
#define PROF_CHK(slot)
#endif

constexpr int kQpThreads = 256;
constexpr int kQpThreadsC = 256;  // (usable in __host__ __device__ constant expressions)
constexpr double kOsqpInf = 1e30;
constexpr double kMinScaling = 1e-4, kMaxScaling = 1e4;
constexpr double kVerifyTol = 1e-9;  // KKT verification of the polished point (deviation D2)
constexpr int kVerifyRounds = 3;
constexpr double kRhoMin = 1e-6, kRhoMax = 1e6, kRhoTol = 1e-4, kRhoEqOverIneq = 1e3;
enum { QPS_UNSOLVED = 0, QPS_SOLVED = 1, QPS_SOLVED_INACC = 2, QPS_PINF = 3, QPS_PINF_INACC = 4, QPS_DINF = 5,
       QPS_DINF_INACC = 6, QPS_MAXITER = 7, QPS_NONCVX = 8 };

__device__ __forceinline__ double limit_scaling(double v) {
  v = v < kMinScaling ? 1.0 : v;
  return v > kMaxScaling ? kMaxScaling : v;
}

// ---- shared memory layout (doubles) ------------------------------------------------------------------
// SA: A_p -> Ainv_p.  SLM: left couplings L_p during the factorisation, Um_p afterwards.  SU: Up_p (while a
// level is being eliminated the still unused slot of the left survivor holds a temporary).
struct QpSmem {
  int SA, SLM, SU, beta, x, zb, yb, v1, w, qs, lbs, ubs, Dz, v2, Pb, tmp, red, colptr, colent, rints, rows, total, row_cap;
  int factor_smem, pband_smem;  // 1: lives in shared memory; 0: in global memory (factor: per-CTA region, band: the shared table)
  int pinv;                     // 1: the factor region also holds the partition-inverse form of the ADMM system (PinvPlan)
};

// ---- partition-inverse form of the block-tridiagonal system (the ADMM system of short trajectories) --------------------
// Blocks 3, 7, 11, ... are SEPARATORS, the runs of <= 3 blocks between them PARTITIONS (independent once the separators are
// known).  With A_pp the partitions, C their coupling to the separators, S = A_ss - C' inv(A_pp) C:
//   factor:  PI = inv(A_pp) (dense, <= 3 NB square per partition);  W = PI C (2 NB columns per partition: its left and its
//            right separator);  Sinv;  Z = [-Sinv W' | Sinv] = the separator rows of the inverse of the whole matrix
//   solve:   step A   y = PI b_p (one thread per partition row, its row of PI in REGISTERS for a whole block of iterations)
//                     x_s = Z b  (two threads per separator row, Z in shared memory)          -- independent of each other
//            step B   x_p = y - W [x_left; x_right]
// Two dependent steps instead of the 2 log2(M) + 1 of the cyclic reduction (7 at 15 blocks), and 8.8 k instead of 26 k
// doubles read from shared memory per solve.  scripts/probes/pinv_proto.py checks the algebra against a dense solve.
// Thread roles: tid < PR owns partition row tid (partition tid / 3NB); PR <= tid < PR + 2 nS: separator row (tid - PR) / 2,
// half (tid - PR) & 1 of its columns.
struct PinvPlan {
  int ok;          // the system fits this path (roles <= 256 threads, <= 3 separators)
  int Ns, nS;      // separator blocks, their rows Ns * NB
  int PR;          // partition rows (M - Ns) * NB
  int ZS, HO;      // row stride of Z (>= Np, = 4 mod 16: the 8 lanes of a quarter warp hit 8 different 16-byte bank groups),
                   // first column of the second half of a separator row (= 2 mod 16, same reason)
  int WS;          // row stride of W (2 NB + 2: consecutive rows 16 bytes apart modulo 128)
  int SS;          // row stride of S / Sinv
  int zo, wo, so;  // offsets (doubles from the start of the factor region) of Z, W, S
  int total;       // doubles of the factor region this path needs
};
__host__ __device__ inline PinvPlan pinv_plan(int M, int nb) {
  PinvPlan pl;
  pl.Ns = M / 4;
  pl.nS = pl.Ns * nb;
  pl.PR = (M - pl.Ns) * nb;
  const int Np = M * nb, blk = nb * nb;
  pl.ok = (nb % 2 == 0) && nb <= 14 && pl.Ns <= 3 && pl.PR + 2 * pl.nS <= 256;
  pl.ZS = Np + ((4 - Np % 16) + 16) % 16;
  pl.HO = ((Np / 2 + 6) / 16) * 16 + 2;
  if (pl.HO > Np) pl.HO = Np;
  pl.WS = 2 * nb + 2;
  pl.SS = pl.nS + (pl.nS & 1);
  const int fA = (M * blk + 15) & ~15, fL = fA + 8, fU = (M * blk + 1) & ~1;
  const int zn = pl.nS * pl.ZS;
  pl.zo = 0;
  // W is written while SA / SLM are still read (Z replaces them at the end), and it sits beyond the whole cyclic-reduction
  // layout: a polish factors its own system there, and a polish that fails hands the ADMM system back without a new
  // factorisation (Z comes back from a copy in global memory, W and the rows of PI were never touched)
  pl.wo = ((zn > fA + fL + fU ? zn : fA + fL + fU) + 15) & ~15;
  pl.so = pl.wo + ((pl.PR * pl.WS + 1) & ~1);
  pl.total = pl.so + pl.nS * pl.SS;
  return pl;
}
constexpr int kQpSmemBudget = 28800;  // doubles per CTA (225 KB of the 227 KB a CTA may use): one CTA per SM
__host__ __device__ inline int qp_block_count(int N, int nb) { return (N + nb - 1) / nb; }
__host__ __device__ inline int qp_even(int v) { return (v + 1) & ~1; }
__host__ __device__ inline int qp_factor_doubles(int N, int nb) { return 3 * qp_even(qp_block_count(N, nb) * nb * nb); }
// per resident CTA in global memory: the factor of wide blocks or the rows of the partition inverses, then the copy of Z
// that survives a polish
__host__ __device__ inline size_t qp_cta_global_doubles(int N, int nb) {
  const PinvPlan pl = pinv_plan(qp_block_count(N, nb), nb);
  return static_cast<size_t>(qp_factor_doubles(N, nb)) + static_cast<size_t>(pl.nS) * pl.ZS;
}
__host__ __device__ inline QpSmem qp_smem_layout(int N, int nb, int row_stride, int CN, int max_rows, bool factor_global) {
  const int M = qp_block_count(N, nb), Np = M * nb, blk = nb * nb;
  QpSmem s;
  int o = 0;
  s.beta = o; o += qp_even(Np);
  s.x = o;    o += qp_even(Np);
  s.zb = o;   o += qp_even(Np);
  s.yb = o;   o += qp_even(Np);
  s.v1 = o;   o += qp_even(Np);
  s.w = o;    o += qp_even(Np);
  s.qs = o;   o += qp_even(Np);
  s.lbs = o;  o += qp_even(Np);
  s.ubs = o;  o += qp_even(Np);
  s.Dz = o;   o += qp_even(Np);
  s.v2 = o;   o += qp_even(Np);
  s.tmp = o;  o += 2 * kQpThreadsC + 64 + 8;          // Gauss-Jordan pivot rows (and column scales), 8 scalars at the end
  s.red = o;  o += 16 * 8;                            // block reductions: 16 quantities x 8 warps
  s.colptr = o; o += qp_even((Np + 2) / 2 + 1);
  // the factor (SA, SLM, SU contiguous) when it fits, then the objective's band P(i, i-k), then rows with what is left
  // (bank layout: the solve reads SA and SU side by side in its backward tasks and SU and SLM side by side in its
  // forward tasks, even lanes one matrix, odd lanes the other: SLM starts a multiple of 16 doubles after SA and SU
  // 8 doubles (16 banks) off that grid, so the two halves of a warp's access land on disjoint banks; before this layout
  // bank conflicts dominated the solve.)
  const int fA = (M * blk + 15) & ~15, fL = fA + 8, fU = qp_even(M * blk);
  s.factor_smem = (!factor_global && o + fA + fL + fU <= kQpSmemBudget) ? 1 : 0;
  o = s.factor_smem ? ((o + 15) & ~15) : o;
  const int per_row2 = 2 * row_stride + CN + RI_NINTS;  // in half doubles: record + column entries + row ints
  // the partition-inverse form needs a larger region (Z, W, S): taken when the band still fits and at least 64 rows
  // (or every row the problem can have) stay on chip
  const PinvPlan pl = pinv_plan(M, nb);
  {
    const int region = qp_even(pl.total > fA + fL + fU ? pl.total : fA + fL + fU);
    const int o2 = o + region + qp_even(N * (nb + 1));
    const int cap2 = (o2 < kQpSmemBudget) ? 2 * (kQpSmemBudget - o2) / per_row2 - 1 : 0;
    s.pinv = (s.factor_smem && pl.ok && cap2 >= (max_rows < 64 ? max_rows : 64)) ? 1 : 0;
  }
  s.SA = o;   o += s.factor_smem ? fA : 0;
  s.SLM = o;  o += s.factor_smem ? fL : 0;
  s.SU = o;   o += s.factor_smem ? fU : 0;
  if (s.pinv && s.SA + pl.total > o) o = s.SA + qp_even(pl.total);
  s.pband_smem = (o + qp_even(N * (nb + 1)) <= kQpSmemBudget) ? 1 : 0;
  s.Pb = o;   o += s.pband_smem ? qp_even(N * (nb + 1)) : 0;
  int cap = (o < kQpSmemBudget) ? 2 * (kQpSmemBudget - o) / per_row2 - 1 : 0;
  cap = cap > max_rows ? max_rows : cap;
  cap = cap > 1023 ? 1023 : cap;
  cap = cap < 0 ? 0 : cap;
  s.row_cap = cap;
  s.colent = o; o += qp_even((cap * CN + 1) / 2);
  s.rints = o;  o += qp_even((cap * RI_NINTS + 1) / 2);
  s.rows = o;   o += cap * row_stride;
  s.total = o;
  return s;
}

// ---- per-row record (global memory): CN raw coefficients, CN scaled coefficients, then these fields ----
// Every row is padded to CN coefficients (zeros) and two aux slots (absent aux: u = b = qa = 0, scalings 1).
enum RowF {
  R_C = 0, R_W,                         // raw: constant, aux cost
  R_E, R_DA0, R_DA1, R_EA0, R_EA1,      // Ruiz scalings
  R_U0, R_U1, R_B0, R_B1, R_LO, R_UP, R_QA0, R_QA1, R_RHO,  // scaled view (R_RHO: 1 = equality row)
  R_XA0, R_XA1, R_Z, R_Y, R_ZA0, R_ZA1, R_YA0, R_YA1,        // ADMM state
  R_RA0, R_RA1, R_COEF, R_WR, R_G0, R_G1, R_DEN, R_WRR,      // per-solve temporaries (WRR: raw row weight)
  R_IDEN, R_IWRR,                                            // reciprocals of DEN / WRR (0 when WRR == 0)
  R_DY, R_DYA0, R_DYA1, R_DXA0, R_DXA1,
  R_PW, R_PWA0, R_PWA1, R_PB, R_PY, R_PYA0, R_PYA1, R_PX0, R_PX1,  // polish
  R_MV,
  R_NF
};
// record = CN raw coefficients | CN scaled coefficients | R_NF fields | CN contributions as[k] * R_COEF of the
// row to the right-hand side of the next ADMM solve
__host__ __device__ inline int qp_row_stride(int CN) { return 3 * CN + R_NF; }

// A vector of the CTA's dynamic shared memory, kept as its offset: q.x[i] is sm[off + i], which the compiler can prove
// to be a shared-memory access (ld.shared / st.shared, and no aliasing with the global-memory stores around it), while a
// plain double* member read back from the context is a generic pointer.  Converts to double* where one is asked for.
struct SmVec {
  int off;
  __device__ __forceinline__ double* ptr() const {
    extern __shared__ double sm[];
    return sm + off;
  }
  __device__ __forceinline__ double& operator[](int i) const { return ptr()[i]; }
  __device__ __forceinline__ operator double*() const { return ptr(); }
  __device__ __forceinline__ SmVec& operator=(double* p) {
    extern __shared__ double sm[];
    off = static_cast<int>(p - sm);
    return *this;
  }
};

struct QpCtx {
  int N, Np, nb, M, T, D, CN, RS, tid, nrows;
  double *SA, *SLM, *SU;                                                 // the factor: shared, or global (wide blocks)
  SmVec beta, x, zb, yb, v1, w, qs, lbs, ubs, tmp, red, flag;            // shared (flag: 8 scalars)
  int* colptr;           // shared [Np+1]
  SmVec Dz, v2;          // shared [Np]: variable scalings, scratch of the residual / polish passes
  double* rows;          // shared when the QP has at most row_cap rows, else global
  double* soa;           // this CTA's block of global memory for the column-major copy of the rows (admm_block_soa)
  double* smbase;        // start of the CTA's dynamic shared memory (generic address), rows_smem: q.rows lives there
  int rows_smem;
  int* rints;
  const int* colent;     // entries: (row << 5) | k (shared or global, like the rows)
  const double* Pband;   // shared copy of the objective band [N][2D+1]
  const int* band_offs;  // the band offsets k with a structurally non-zero P(i, i-k), ascending; n_band of them
  int n_band;
  double* scratch;
  int pinv;              // the ADMM system is factored in its partition-inverse form (pl)
  PinvPlan pl;
  double* pi_g;          // this CTA's block of global memory for the rows of the partition inverses, column-major
                         // [3 NB][PR]: a warp's loads and stores of one column are contiguous
  double* z_stash;       // ... and for the copy of Z taken before a polish
  double c, cinv, rho, rho_eq, sigma, alpha;
  __device__ __forceinline__ double* R(int r) const { return rows + static_cast<size_t>(r) * RS; }
  __device__ __forceinline__ double* F(int r) const { return rows + static_cast<size_t>(r) * RS + 2 * CN; }
  __device__ __forceinline__ const int* I(int r) const { return rints + static_cast<size_t>(r) * RI_NINTS; }
};

// ---- block reductions: inside each warp, then 8 partials through shared memory ------------------------------
// vals[k] -> max, or (bit k of sum_mask set) the sum; fixed order, every thread gets the result.  Every quantity that
// is max-reduced here is a norm (>= 0, built from fabs): non-negative doubles order like their bit patterns, so the
// warp maximum is two 32-bit redux instructions (high word, then the low words of the lanes that hold it) instead of
// five 64-bit shuffle steps.  NaNs are ignored, as fmax ignores them.
__device__ __forceinline__ double warp_max_norm(double v) {
  v = (v != v) ? 0.0 : v;
  const unsigned hi = static_cast<unsigned>(__double2hiint(v)) & 0x7fffffffu, lo = static_cast<unsigned>(__double2loint(v));
  const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
  const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
  return __hiloint2double(static_cast<int>(mh), static_cast<int>(ml));
}
template <int NQ, unsigned SUM_MASK>
__device__ __forceinline__ void block_reduce(const QpCtx& q, double (&vals)[NQ]) {
  static_assert(NQ <= 16, "red area too small");
  // (forced inline with compile-time roles: the values stay in registers; the partials go through shared-memory
  // offsets, not generic pointers)
  extern __shared__ double sm[];
  double* const red = sm + (q.red - q.smbase);
  const int lane = q.tid & 31, wid = q.tid >> 5;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < NQ; ++k) {
    double v = vals[k];
    if ((SUM_MASK >> k) & 1u) {  // (a constant once the loop is unrolled)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    } else {
      v = warp_max_norm(v);
    }
    vals[k] = v;
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < NQ; ++k) red[k * 8 + wid] = vals[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NQ; ++k) {
    if ((SUM_MASK >> k) & 1u) {  // (a constant once the loop is unrolled)
      double acc = red[k * 8];
#pragma unroll
      for (int w = 1; w < kQpThreads / 32; ++w) acc += red[k * 8 + w];
      vals[k] = acc;
    } else {
      vals[k] = warp_max_norm(red[k * 8 + (lane & 7)]);  // every warp reduces the 8 partials again
    }
  }
  __syncthreads();
}

// weights of the linear system: ADMM (rho vector, sigma) or polish (1/delta on the active set, delta)
struct SysW {
  bool polish;
  double sig, rho_aux;
#ifdef TB200_PROFILE
  int prof_kind = 0;  // the profiler slots of assemble_factor: 0 the initial factorisation, 1 a later one (polish: 2)
#endif
};

// variable index of coefficient k of a row (padding coefficients alias the last real one; their value is 0)
__device__ __forceinline__ int row_var(const int* I, int k) {
  return I[RI_BASE] + min(k, I[RI_CNT] - 1) * I[RI_STRIDE];
}

// ---------------------------------------------------------------------------------------------------
// Block cyclic reduction: factorisation.  On entry SA[p] = K(p,p), SLM[p] = K(p,p-1) (p >= 1).  On exit
// SA[p] = Ainv_p, SLM[p] = Um_p, SU[p] = Up_p for the level at which block p is eliminated.
// One thread owns one matrix row (NB doubles in registers) in every phase; rows of the other operand are read
// from shared memory as 16-byte broadcasts.
template <int NB>
__device__ __forceinline__ void load_row(double (&a)[NB], const double* src) {
  const double2* s2 = reinterpret_cast<const double2*>(src);
#pragma unroll
  for (int k = 0; k < NB / 2; ++k) {
    const double2 v = s2[k];
    a[2 * k] = v.x;
    a[2 * k + 1] = v.y;
  }
}
template <int NB>
__device__ __forceinline__ void store_row(double* dst, const double (&a)[NB]) {
  double2* d2 = reinterpret_cast<double2*>(dst);
#pragma unroll
  for (int k = 0; k < NB / 2; ++k) d2[k] = make_double2(a[2 * k], a[2 * k + 1]);
}
// out[j] (+)= sum_k x[k] * Y[k][j]   (x in registers, Y row major in shared memory)
template <int NB>
__device__ __forceinline__ void row_times_mat(double (&out)[NB], const double (&x)[NB], const double* Y) {
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    double y[NB];
    load_row<NB>(y, Y + k * NB);
#pragma unroll
    for (int j = 0; j < NB; ++j) out[j] += x[k] * y[j];
  }
}
// out[j] (+)= sum_k x[k] * Y[j][k]   (x times Y transposed)
template <int NB>
__device__ __forceinline__ void row_times_matT(double (&out)[NB], const double (&x)[NB], const double* Y) {
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    double y[NB];
    load_row<NB>(y, Y + j * NB);
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int k = 0; k < NB; k += 2) {
      a0 += x[k] * y[k];
      a1 += x[k + 1] * y[k + 1];
    }
    out[j] += a0 + a1;
  }
}
// WARP (blocks of <= 16 with the factor in shared memory): every block is inverted by one half warp, lanes 0..NB-1 of
// the half holding its rows, so the steps of an inversion synchronise that warp only; the factor is addressed as
// shared memory.  Otherwise the blocks of a chunk lie side by side over the CTA and every step is a CTA barrier.  Both
// compute every value by the same expression in the same order.
template <int NB, bool WARP>
__device__ inline bool bcr_factor(const QpCtx& q) {
  static_assert(!WARP || NB <= 16, "a block per half warp");
  constexpr int BLK = NB * NB, G = kQpThreads / 2;  // two thread groups work side by side where possible
  // blocks per task chunk: inversion (all threads) / products (per group)
  constexpr int CH1 = WARP ? kQpThreads / 16 : kQpThreads / NB, CH2 = G / NB;
  extern __shared__ double sm[];
  double* const SA = WARP ? sm + (q.SA - q.smbase) : q.SA;
  double* const SLM = WARP ? sm + (q.SLM - q.smbase) : q.SLM;
  double* const SU = WARP ? sm + (q.SU - q.smbase) : q.SU;
  const int M = q.M, tid = q.tid;
  const int grp = tid >= G, gt = tid - (grp ? G : 0);
  int bad = 0;
  for (int l = 0; (1 << l) - 1 < M; ++l) {
    const int s = 1 << l, first = s - 1, sh = l + 1;  // eliminated p = first + (e << sh); survivors j = p + s
    const int nE = (M + s) >> sh, nS = M >> sh;
    PROF_T0();
    // ---- 1. Ainv_p in place: Gauss-Jordan without pivoting (the blocks are symmetric positive definite);
    //         thread (e,i) keeps row i of block e in registers, the pivot row goes through shared memory
    for (int e0 = 0; e0 < nE; e0 += CH1) {
      const int nc = (nE - e0 < CH1) ? nE - e0 : CH1;
      const int e = WARP ? tid >> 4 : tid / NB, i = WARP ? tid & 15 : tid % NB;
      const bool act = WARP ? (i < NB && e < nc) : tid < nc * NB;
      double* A = SA + (first + ((e0 + (act ? e : 0)) << sh)) * BLK + (act ? i : 0) * NB;
      double a[NB];
      load_row<NB>(a, A);
#pragma unroll
      for (int k = 0; k < NB; ++k) {
        double* prow = q.tmp + (k & 1) * (CH1 * NB) + e * NB;  // (double buffered: one barrier per step)
        if (act && i == k) {
          const double piv = a[k];
          if (!(piv > 0.0)) bad = 1;
          const double ip = 1.0 / piv;
#pragma unroll
          for (int j = 0; j < NB; ++j) a[j] = (j == k) ? ip : a[j] * ip;
          store_row<NB>(prow, a);
        }
        if constexpr (WARP) __syncwarp();
        else __syncthreads();
        if (act && i != k) {
          double pr[NB];
          load_row<NB>(pr, prow);
          const double f = a[k];
#pragma unroll
          for (int j = 0; j < NB; ++j) a[j] = (j == k) ? -f * pr[k] : a[j] - f * pr[j];
        }
      }
      if (act) store_row<NB>(A, a);
    }
    __syncthreads();
    PROF_ADD(30);  // (the inversions of every level, all factorisations by the cyclic reduction)
    // ---- 2. group 0: Up_p = L_{p+s} Ainv_p -> SU[p];  group 1: Um_p = L_p' Ainv_p -> SU[p-s] (temporary home)
    for (int e0 = 0; e0 < nE; e0 += CH2) {
      const int nc = (nE - e0 < CH2) ? nE - e0 : CH2;
      const bool act = gt < nc * NB;
      const int e = e0 + (act ? gt / NB : 0), i = gt % NB;
      const int p = first + (e << sh);
      const double* Ai = SA + p * BLK;
      if (act && grp == 0 && p + s < M) {
        double x[NB], out[NB];
        load_row<NB>(x, SLM + (p + s) * BLK + i * NB);
#pragma unroll
        for (int j = 0; j < NB; ++j) out[j] = 0.0;
        row_times_mat<NB>(out, x, Ai);
        store_row<NB>(SU + p * BLK + i * NB, out);
      }
      if (act && grp == 1 && p - s >= 0) {
        double x[NB], out[NB];
        const double* L = SLM + p * BLK + i;  // column i of L_p
#pragma unroll
        for (int k = 0; k < NB; ++k) x[k] = L[k * NB];
#pragma unroll
        for (int j = 0; j < NB; ++j) out[j] = 0.0;
        row_times_mat<NB>(out, x, Ai);
        store_row<NB>(SU + (p - s) * BLK + i * NB, out);
      }
    }
    __syncthreads();
    // ---- 3./4. survivors j = p + s.  group 0: A_j -= Up_{j-s} L_j', and L'_j = -Up_{j-s} L_{j-s} (kept in registers);
    //            group 1: t2 = Um_{j+s} L_{j+s} (Um_{j+s} sits in SU[j]), subtracted from A_j after the barrier.
    //            (A chunk only writes blocks of its own survivors, which no other chunk reads: no barrier between chunks.)
    for (int e0 = 0; e0 < nS; e0 += CH2) {
      const int nc = (nS - e0 < CH2) ? nS - e0 : CH2;
      const bool act = gt < nc * NB;
      const int e = e0 + (act ? gt / NB : 0), i = gt % NB;
      const int j = first + s + (e << sh), p = j - s;
      double keep[NB];
#pragma unroll
      for (int c = 0; c < NB; ++c) keep[c] = 0.0;
      if (act && grp == 0) {
        double x[NB], t1[NB];
        load_row<NB>(x, SU + p * BLK + i * NB);  // row i of Up_p
#pragma unroll
        for (int c = 0; c < NB; ++c) t1[c] = 0.0;
        row_times_matT<NB>(t1, x, SLM + j * BLK);
        if (p - s >= 0) row_times_mat<NB>(keep, x, SLM + p * BLK);
        double arow[NB];
        load_row<NB>(arow, SA + j * BLK + i * NB);
#pragma unroll
        for (int c = 0; c < NB; ++c) arow[c] -= t1[c];
        store_row<NB>(SA + j * BLK + i * NB, arow);
      }
      if (act && grp == 1 && j + s < M) {
        double x[NB];
        load_row<NB>(x, SU + j * BLK + i * NB);  // row i of Um_{j+s}
        row_times_mat<NB>(keep, x, SLM + (j + s) * BLK);
      }
      __syncthreads();
      if (act && grp == 0) {
#pragma unroll
        for (int c = 0; c < NB; ++c) keep[c] = -keep[c];
        store_row<NB>(SLM + j * BLK + i * NB, keep);  // new left coupling (0 without a left survivor)
      }
      if (act && grp == 1 && j + s < M) {
        double arow[NB];
        load_row<NB>(arow, SA + j * BLK + i * NB);
#pragma unroll
        for (int c = 0; c < NB; ++c) arow[c] -= keep[c];
        store_row<NB>(SA + j * BLK + i * NB, arow);
      }
    }
    __syncthreads();
    // ---- 5. Um_p moves from its temporary home into SLM[p] (L_p is dead now)
    for (int t = tid; t < nE * BLK; t += kQpThreads) {
      const int e = t / BLK, r = t % BLK;
      const int p = first + (e << sh);
      if (p - s >= 0) SLM[p * BLK + r] = SU[(p - s) * BLK + r];
    }
    __syncthreads();
  }
  // every thread must agree on the verdict
  if (tid == 0) q.flag[0] = 0.0;
  __syncthreads();
  if (bad) q.flag[0] = 1.0;
  __syncthreads();
  const bool ok = q.flag[0] == 0.0;
  __syncthreads();
  return ok;
}

// Block cyclic reduction: solve K w = v (both in shared memory, length Np; v is overwritten by the reduced
// right-hand sides).  Two threads per (block,row) task, combined with one shuffle; every level ends in a barrier.
template <int NB>
__device__ __forceinline__ double dot_row(const double* __restrict__ m, const double* __restrict__ v) {
  const double2* m2 = reinterpret_cast<const double2*>(m);
  const double2* v2 = reinterpret_cast<const double2*>(v);
  double a0 = 0.0, a1 = 0.0;
#pragma unroll
  for (int k = 0; k < NB / 2; ++k) {
    const double2 mm = m2[k], vv = v2[k];
    a0 += mm.x * vv.x;
    a1 += mm.y * vv.y;
  }
  return a0 + a1;
}
template <int NB>
__device__ inline void bcr_solve(const QpCtx& q, double* v, double* w) {
  constexpr int BLK = NB * NB, H = NB / 2;
  const int M = q.M, tid = q.tid, side = tid & 1, task0 = tid >> 1;
  __syncthreads();
  int l = 0;
  // ---- down: survivors absorb their eliminated neighbours
  for (; (2 << l) - 1 < M; ++l) {
    const int s = 1 << l, sh = l + 1, nS = M >> sh;
    for (int tb = 0; tb < nS * NB; tb += kQpThreads / 2) {
      if (tb + ((tid & ~31) >> 1) >= nS * NB) continue;  // warp-uniform: this warp has no task in this chunk
      const int task = tb + task0;
      const int e = task / NB, r = task % NB;
      const bool act = e < nS;
      const int j = 2 * s - 1 + ((act ? e : 0) << sh);
      const int pb = side ? j + s : j - s;           // side 0: left eliminated neighbour, side 1: right one
      const bool valid = act && pb < M;
      const int pbc = valid ? pb : j - s;
      const double* mat = (side ? q.SLM : q.SU) + pbc * BLK + r * NB;
      double a = dot_row<NB>(mat, v + pbc * NB);
      a = valid ? a : 0.0;
      const double o = __shfl_xor_sync(0xffffffffu, a, 1);
      if (act && side == 0) v[j * NB + r] -= a + o;  // survivors are not read by any other task of this level
    }
    __syncthreads();
  }
  // ---- up: eliminated blocks, from the last level back to the first
  for (; l >= 0; --l) {
    const int s = 1 << l, first = s - 1, sh = l + 1;
    if (first >= M) continue;
    const int nE = (M + s) >> sh;
    for (int tb = 0; tb < nE * NB; tb += kQpThreads / 2) {
      if (tb + ((tid & ~31) >> 1) >= nE * NB) continue;  // warp-uniform: this warp has no task in this chunk
      const int task = tb + task0;
      const int e = task / NB, r = task % NB;
      const bool act = e < nE;
      const int p = first + ((act ? e : 0) << sh);
      const bool hasl = p - s >= 0, hasr = p + s < M;
      // both sides run the same instruction stream: a column dot of length NB plus half of the Um column dot
      //   side 0:  +Ainv_p(:,r) . v_p        - Um_p(0:H,r) . w_{p-s}(0:H)      (Ainv is symmetric)
      //   side 1:  -Up_p(:,r)   . w_{p+s}    - Um_p(H:NB,r) . w_{p-s}(H:NB)
      const double* X = (side ? q.SU : q.SA) + p * BLK + r;
      const double* y = side ? w + (hasr ? p + s : 0) * NB : v + p * NB;
      const double* Um = q.SLM + p * BLK + (side ? H * NB : 0) + r;
      const double* wl = w + (hasl ? p - s : 0) * NB + (side ? H : 0);
      double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll
      for (int k = 0; k < NB; k += 2) {
        a0 += X[k * NB] * y[k];
        a1 += X[(k + 1) * NB] * y[k + 1];
      }
#pragma unroll
      for (int k = 0; k < H; ++k) a2 += Um[k * NB] * wl[k];
      const double dx = a0 + a1;
      const double acc = (side ? (hasr ? -dx : 0.0) : dx) - (hasl ? a2 : 0.0);
      const double o = __shfl_xor_sync(0xffffffffu, acc, 1);
      if (act && side == 0) w[p * NB + r] = acc + o;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------
// Fixed per-thread roles in the solve (bcr_solve_hyb, bcr_solve_sm), computed once per block.  The factor does not
// change between two refactorisations, and every thread applies the same few matrix rows in every solve: level 0 gives
// each thread one forward row (NB doubles) and one backward row (NB + NB/2), and the upper levels are spread over
// the threads so that nobody owns more than one upper forward and one upper backward row.
struct SolveRoles {
  int n_fwd, n_lvl;                       // forward levels, all levels (the last ones only go up)
  int f0_warps, b0_warps;                 // thread ranges (rounded up to warps) with level-0 work
  int f0_vec, f0_dst, b0_y, b0_wl, b0_dst;
  int fu_level, fu_vec, fu_dst, bu_level, bu_y, bu_wl, bu_dst;
  bool f0_valid, f0_store, b0_store, b0_hasl, b0_hasr, b0_yw;
  bool fu_valid, fu_store, bu_store, bu_hasl, bu_hasr, bu_yw;  // *_yw: the NB-long operand is read from w, not v
  // upper-level rows read from the factor in shared memory (bcr_solve_hyb): offsets in doubles from the start of the
  // dynamic shared memory, valid when the factor lives there
  int fu_mat, bu_X, bu_Um, f0_mat, b0_X, b0_Um;
};
template <int NB>
__device__ inline SolveRoles solve_roles(const QpCtx& q) {
  SolveRoles R{};
  const int M = q.M, tid = q.tid;
  int nf = 0;
  while ((2 << nf) - 1 < M) ++nf;
  int nl = 0;
  while ((1 << nl) - 1 < M) ++nl;
  R.n_fwd = nf;
  R.n_lvl = nl;
  constexpr int BLK = NB * NB;
  const int oSA = static_cast<int>(q.SA - q.smbase), oSLM = static_cast<int>(q.SLM - q.smbase), oSU = static_cast<int>(q.SU - q.smbase);
  auto fwd_role = [&](int l, int u, int& vec, int& dst, bool& valid, bool& store) {
    const int s = 1 << l, sh = l + 1, nS = M >> sh;
    const int task = u >> 1, side = u & 1, e = task / NB, r = task % NB;
    const bool act = e < nS;
    const int j = 2 * s - 1 + ((act ? e : 0) << sh);
    const int pb = side ? j + s : j - s;
    valid = act && pb < M;
    vec = (valid ? pb : j - s) * NB;
    dst = j * NB + r;
    store = act && side == 0;
    (l > 0 ? R.fu_mat : R.f0_mat) = (side ? oSLM : oSU) + (valid ? pb : j - s) * BLK + r * NB;
  };
  auto bwd_role = [&](int l, int u, int& y, int& wl, int& dst, bool& store, bool& hasl, bool& hasr, bool& yw) {
    const int s = 1 << l, first = s - 1, sh = l + 1, nE = (M + s) >> sh;
    const int task = u >> 1, side = u & 1, e = task / NB, r = task % NB;
    const bool act = e < nE;
    const int p = first + ((act ? e : 0) << sh);
    hasl = p - s >= 0;
    hasr = p + s < M;
    yw = side;
    y = side ? (hasr ? p + s : 0) * NB : p * NB;
    wl = (hasl ? p - s : 0) * NB + (side ? NB / 2 : 0);
    dst = p * NB + r;
    store = act && side == 0;
    (l > 0 ? R.bu_X : R.b0_X) = (side ? oSU : oSA) + p * BLK + r;
    (l > 0 ? R.bu_Um : R.b0_Um) = oSLM + p * BLK + (side ? (NB / 2) * NB : 0) + r;
  };
  // level 0: thread = (task, side)
  fwd_role(0, tid, R.f0_vec, R.f0_dst, R.f0_valid, R.f0_store);
  R.f0_warps = (2 * (M >> 1) * NB + 31) & ~31;
  bwd_role(0, tid, R.b0_y, R.b0_wl, R.b0_dst, R.b0_store, R.b0_hasl, R.b0_hasr, R.b0_yw);
  R.b0_warps = (2 * ((M + 1) >> 1) * NB + 31) & ~31;
  // upper levels: consecutive thread ranges (even offsets keep the (u, u^1) pairs inside a warp)
  R.fu_level = -1;
  R.bu_level = -1;
  int off = 0;
  for (int l = 1; l < nf; ++l) {
    const int cnt = 2 * (M >> (l + 1)) * NB;
    if (tid >= off && tid < off + cnt) {
      R.fu_level = l;
      fwd_role(l, tid - off, R.fu_vec, R.fu_dst, R.fu_valid, R.fu_store);
    }
    off += cnt;
  }
  off = 0;
  for (int l = 1; l < nl; ++l) {
    const int cnt = 2 * ((M + (1 << l)) >> (l + 1)) * NB;
    if (tid >= off && tid < off + cnt) {
      R.bu_level = l;
      bwd_role(l, tid - off, R.bu_y, R.bu_wl, R.bu_dst, R.bu_store, R.bu_hasl, R.bu_hasr, R.bu_yw);
    }
    off += cnt;
  }
  return R;
}
// true when the upper-level roles fit the CTA (host-checked as well)
__host__ __device__ inline bool solve_roles_fit(int M, int NB) {
  int f = 0, b = 0;
  for (int l = 1; (2 << l) - 1 < M; ++l) f += 2 * (M >> (l + 1)) * NB;
  for (int l = 1; (1 << l) - 1 < M; ++l) b += 2 * ((M + (1 << l)) >> (l + 1)) * NB;
  return f <= kQpThreads && b <= kQpThreads && 2 * ((M + 1) >> 1) * NB <= kQpThreads;
}
// the thread's backward matrix row, from the factor in shared memory
template <int NB>
__device__ __forceinline__ void load_bwd_row(const QpCtx& q, int l, int u, double (&m)[NB + NB / 2]) {
  constexpr int BLK = NB * NB, H = NB / 2;
  const int M = q.M, s = 1 << l, first = s - 1, sh = l + 1, nE = (M + s) >> sh;
  const int task = u >> 1, side = u & 1, e = task / NB, r = task % NB;
  const bool act = e < nE;
  const int p = first + ((act ? e : 0) << sh);
  const double* X = (side ? q.SU : q.SA) + p * BLK + r;
  const double* Um = q.SLM + p * BLK + (side ? H * NB : 0) + r;
#pragma unroll
  for (int k = 0; k < NB; ++k) m[k] = act ? X[k * NB] : 0.0;
#pragma unroll
  for (int k = 0; k < H; ++k) m[NB + k] = act ? Um[k * NB] : 0.0;
}

// Shared-memory loads that stay where they are written: every level of the solve is a short dependent chain (loads ->
// 14 multiply-adds -> shuffle -> store -> barrier), and a schedule that interleaves one load with the two multiply-adds
// that consume it exposes the load latency seven times per level instead of once.
__device__ __forceinline__ double2 lds_v2(const double* p) {
  double2 v;
  const unsigned a = static_cast<unsigned>(__cvta_generic_to_shared(p));
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a));
  return v;
}
// ... from a 32-bit shared-memory address computed once (base + constant folds into the load's immediate offset)
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ double2 lds_v2_at(const unsigned a) {
  double2 v;
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ double lds_f64(const double* p) {
  double v;
  const unsigned a = static_cast<unsigned>(__cvta_generic_to_shared(p));
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
  return v;
}
// Solve for the ADMM block with every level reading its factor rows from shared memory through fixed per-thread
// roles (offsets computed once per block).  No matrix row is kept in a register: the block's register budget goes to
// having all the loads of a level in flight at once.
template <int NB>
__device__ __forceinline__ double bcr_fwd_task(const double* mrow, const double* yv) {
  constexpr int H = NB / 2;
  double2 mm[H], yy[H];
#pragma unroll
  for (int k = 0; k < H; ++k) {
    mm[k] = lds_v2(mrow + 2 * k);
    yy[k] = lds_v2(yv + 2 * k);
  }
  double a0 = 0.0, a1 = 0.0;
#pragma unroll
  for (int k = 0; k < H; ++k) {
    a0 += mm[k].x * yy[k].x;
    a1 += mm[k].y * yy[k].y;
  }
  return a0 + a1;
}
template <int NB>
__device__ __forceinline__ double bcr_bwd_task(const double* X, const double* Um, const double* y, const double* wl,
                                               bool side, bool hasl, bool hasr) {
  constexpr int H = NB / 2;
  double2 yy[H];
  double xx[NB], um[H], ww[H];
#pragma unroll
  for (int k = 0; k < H; ++k) yy[k] = lds_v2(y + 2 * k);
#pragma unroll
  for (int k = 0; k < NB; ++k) xx[k] = lds_f64(X + k * NB);
#pragma unroll
  for (int k = 0; k < H; ++k) {
    um[k] = lds_f64(Um + k * NB);
    ww[k] = lds_f64(wl + k);
  }
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll
  for (int k = 0; k < H; ++k) {
    a0 += xx[2 * k] * yy[k].x;
    a1 += xx[2 * k + 1] * yy[k].y;
  }
#pragma unroll
  for (int k = 0; k < H; ++k) a2 += um[k] * ww[k];
  const double dx = a0 + a1;
  return (side ? (hasr ? -dx : 0.0) : dx) - (hasl ? a2 : 0.0);
}
template <int NB>
__device__ __forceinline__ void bcr_solve_sm(const int tid, const SolveRoles& R, const double* sm_base, double* v, double* w) {
  const int wbase = tid & ~31;
  const bool side = tid & 1;
#if defined(TB200_PROFILE) && !defined(TB200_PROFILE_CHECK)
  long long pt_ = clock64();
#define PROF_LVL(slot) do { const long long n_ = clock64(); if (tid == 0) atomicAdd(&g_prof[slot], (unsigned long long)(n_ - pt_)); pt_ = n_; } while (0)
#else
#define PROF_LVL(slot)
#endif
  __syncthreads();
  PROF_LVL(4);   // wait for the right-hand side
  // ---- down
  if (wbase < R.f0_warps) {
    double a = bcr_fwd_task<NB>(sm_base + R.f0_mat, v + R.f0_vec);
    a = R.f0_valid ? a : 0.0;
    const double o = __shfl_xor_sync(0xffffffffu, a, 1);
    if (R.f0_store) v[R.f0_dst] -= a + o;
  }
  __syncthreads();
  PROF_LVL(14);  // level 0 down
  for (int l = 1; l < R.n_fwd; ++l) {
    const bool mine = R.fu_level == l;
    if (__any_sync(0xffffffffu, mine)) {
      double a = bcr_fwd_task<NB>(sm_base + (mine ? R.fu_mat : 0), v + (mine ? R.fu_vec : 0));
      a = (mine && R.fu_valid) ? a : 0.0;
      const double o = __shfl_xor_sync(0xffffffffu, a, 1);
      if (mine && R.fu_store) v[R.fu_dst] -= a + o;
    }
    __syncthreads();
  }
  PROF_LVL(15);  // upper levels down
  // ---- up
  for (int l = R.n_lvl - 1; l >= 1; --l) {
    const bool mine = R.bu_level == l;
    if (__any_sync(0xffffffffu, mine)) {
      double acc = bcr_bwd_task<NB>(sm_base + (mine ? R.bu_X : 0), sm_base + (mine ? R.bu_Um : 0),
                                    (R.bu_yw ? w : v) + (mine ? R.bu_y : 0), w + (mine ? R.bu_wl : 0), R.bu_yw, R.bu_hasl,
                                    R.bu_hasr);
      acc = mine ? acc : 0.0;
      const double o = __shfl_xor_sync(0xffffffffu, acc, 1);
      if (mine && R.bu_store) w[R.bu_dst] = acc + o;
    }
    __syncthreads();
  }
  PROF_LVL(9);   // upper levels up (slot 9 is otherwise the QP-step counter: read before it is used as such)
  if (wbase < R.b0_warps) {
    const double acc = bcr_bwd_task<NB>(sm_base + R.b0_X, sm_base + R.b0_Um, (side ? w : v) + R.b0_y, w + R.b0_wl, side,
                                        R.b0_hasl, R.b0_hasr);
    const double o = __shfl_xor_sync(0xffffffffu, acc, 1);
    if (R.b0_store) w[R.b0_dst] = acc + o;
  }
  __syncthreads();
}

// A backward task with its factor row in registers (called with the whole register file at its disposal): every thread
// applies the same row in every solve, so it is loaded once per block and the task only reads the right-hand side —
// a few distinct 16-byte words per warp — from shared memory.  With the rows read from shared memory instead, level 0
// alone would move 44 KB (down) and 75 KB (up) per solve through the 128 B/clock shared-memory port, 210 KB per solve
// in all = 1640 cycles of pure bandwidth.  The loads are issued before the multiply-adds.
template <int NB>
__device__ __forceinline__ double reg_bwd_task(const double (&m)[NB + NB / 2], const double* y, const double* wl, bool side,
                                               bool hasl, bool hasr) {
  constexpr int H = NB / 2;
  double2 yy[H];
  double ww[H];
#pragma unroll
  for (int k = 0; k < H; ++k) yy[k] = lds_v2(y + 2 * k);
#pragma unroll
  for (int k = 0; k < H; ++k) ww[k] = lds_f64(wl + k);
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll
  for (int k = 0; k < H; ++k) {
    a0 += m[2 * k] * yy[k].x;
    a1 += m[2 * k + 1] * yy[k].y;
  }
#pragma unroll
  for (int k = 0; k < H; ++k) a2 += m[NB + k] * ww[k];
  const double dx = a0 + a1;
  return (side ? (hasr ? -dx : 0.0) : dx) - (hasl ? a2 : 0.0);
}

// The solve of admm_block_fast: the level-0 backward rows (every thread has one: 75 KB of factor rows per solve if they
// were read from shared memory) are held in registers; the level-0 forward rows and the upper levels (a few warps each,
// 91 KB per solve in all) are read from shared memory.  All four row sets in registers (140 registers) do not fit beside
// the loop's own state even with the whole register file.
template <int NB>
__device__ __forceinline__ void bcr_solve_hyb(const int tid, const SolveRoles& R, const double (&mB0)[NB + NB / 2],
                                              const double* sm_base, double* v, double* w) {
  const int wbase = tid & ~31;
  const bool side = tid & 1;
  __syncthreads();
  // ---- down
  if (wbase < R.f0_warps) {
    double a = bcr_fwd_task<NB>(sm_base + R.f0_mat, v + R.f0_vec);
    a = R.f0_valid ? a : 0.0;
    const double o = __shfl_xor_sync(0xffffffffu, a, 1);
    if (R.f0_store) v[R.f0_dst] -= a + o;
  }
  __syncthreads();
  for (int l = 1; l < R.n_fwd; ++l) {
    const bool mine = R.fu_level == l;
    if (__any_sync(0xffffffffu, mine)) {
      double a = bcr_fwd_task<NB>(sm_base + (mine ? R.fu_mat : 0), v + (mine ? R.fu_vec : 0));
      a = (mine && R.fu_valid) ? a : 0.0;
      const double o = __shfl_xor_sync(0xffffffffu, a, 1);
      if (mine && R.fu_store) v[R.fu_dst] -= a + o;
    }
    __syncthreads();
  }
  // ---- up
  for (int l = R.n_lvl - 1; l >= 1; --l) {
    const bool mine = R.bu_level == l;
    if (__any_sync(0xffffffffu, mine)) {
      double acc = bcr_bwd_task<NB>(sm_base + (mine ? R.bu_X : 0), sm_base + (mine ? R.bu_Um : 0),
                                    (R.bu_yw ? w : v) + (mine ? R.bu_y : 0), w + (mine ? R.bu_wl : 0), R.bu_yw, R.bu_hasl,
                                    R.bu_hasr);
      acc = mine ? acc : 0.0;
      const double o = __shfl_xor_sync(0xffffffffu, acc, 1);
      if (mine && R.bu_store) w[R.bu_dst] = acc + o;
    }
    __syncthreads();
  }
  if (wbase < R.b0_warps) {
    const double acc = reg_bwd_task<NB>(mB0, (side ? w : v) + R.b0_y, w + R.b0_wl, side, R.b0_hasl, R.b0_hasr);
    const double o = __shfl_xor_sync(0xffffffffu, acc, 1);
    if (R.b0_store) w[R.b0_dst] = acc + o;
  }
  __syncthreads();
}

// scaled P (band) times a vector: out = c * Dz .* (P (Dz .* in)); in: shared or global, out: global/shared.
// The band loads are independent and fully unrolled, so the pass costs one memory round trip, not 2*HB+1.
// row i < N of that product; Dz and vin are shared-memory vectors
template <int NB>
__device__ __forceinline__ double p_row(const QpCtx& q, const int i, const double* Dz, const double* vin) {
  constexpr int HB = NB, W = HB + 1;
  const int N = q.N, nbo = q.n_band;
  const double* const Pb = q.Pband;  // shared or global
  const int* const offs = q.band_offs;
  double s = 0.0;
  // (P * Dz) and x, multiplied and added in the reference's order: the lower part of row i (k ascending), then the
  // upper part; only the structurally non-zero offsets are visited (a skipped entry adds an exact zero)
  for (int t0 = 0; t0 < nbo; t0 += 4) {
    double v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = (t0 + u < nbo) ? offs[t0 + u] : -1;
      v[u] = (k >= 0 && k <= i) ? (Pb[i * W + k] * Dz[i - k]) * vin[i - k] : 0.0;
    }
    s += v[0]; s += v[1]; s += v[2]; s += v[3];
  }
  for (int t0 = 0; t0 < nbo; t0 += 4) {
    double v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = (t0 + u < nbo) ? offs[t0 + u] : -1;
      v[u] = (k >= 1 && i + k < N) ? (Pb[(i + k) * W + k] * Dz[i + k]) * vin[i + k] : 0.0;
    }
    s += v[0]; s += v[1]; s += v[2]; s += v[3];
  }
  return s * (q.c * Dz[i]);
}
template <int NB>
__device__ __forceinline__ void p_matvec(const QpCtx& q, const double* in, double* out) {
  // in, out and the scalings are vectors of the CTA's shared memory: addressed as offsets (ld.shared); the band
  // offsets are visited four at a time with their loads side by side
  extern __shared__ double sm[];
  const int N = q.N, Np = q.Np;
  const double* const Dz = sm + (q.Dz - q.smbase);
  const double* const vin = sm + (in - q.smbase);
  double* const vout = sm + (out - q.smbase);
  for (int i = q.tid; i < Np; i += kQpThreads) vout[i] = (i < N) ? p_row<NB>(q, i, Dz, vin) : 0.0;
  __syncthreads();
}

// ---- the terms of a termination check, per row and per variable -------------------------------------------
// Shared by the generic passes of qp_solve_block and the check fused into admm_block_pinv, so that both compute every
// term with the same expression.  m[14]: 0 pri 1 z 2 ax 3 dua 4 aty 5 q 6 px | 7..13 the same on the scaled quantities.
__device__ __forceinline__ void info_row_terms(const double* F, const double ax, double (&m)[14]) {
  const double einv = 1.0 / F[R_E];
  m[0] = fmax(m[0], fabs(einv * (ax - F[R_Z])));
  m[1] = fmax(m[1], fabs(einv * F[R_Z]));
  m[2] = fmax(m[2], fabs(einv * ax));
  m[7] = fmax(m[7], fabs(ax - F[R_Z]));
  m[8] = fmax(m[8], fabs(F[R_Z]));
  m[9] = fmax(m[9], fabs(ax));
#pragma unroll
  for (int k = 0; k < 2; ++k) {  // absent aux slots contribute exact zeros
    const double u = F[R_U0 + k], bb = F[R_B0 + k], qa = F[R_QA0 + k];
    const double xa = F[R_XA0 + k], za = F[R_ZA0 + k], ya = F[R_YA0 + k];
    // Einv / Dinv of the aux row and column: one reciprocal each, multiplied like the Einv[r] * (...) of the oracle
    const double iea = 1.0 / F[R_EA0 + k], ida = 1.0 / F[R_DA0 + k];
    const double axb = bb * xa;
    m[0] = fmax(m[0], fabs(iea * (axb - za)));
    m[1] = fmax(m[1], fabs(iea * za));
    m[2] = fmax(m[2], fabs(iea * axb));
    m[7] = fmax(m[7], fabs(axb - za));
    m[8] = fmax(m[8], fabs(za));
    m[9] = fmax(m[9], fabs(axb));
    const double aty = u * F[R_Y] + bb * ya;
    m[3] = fmax(m[3], fabs(ida * (qa + aty)));
    m[4] = fmax(m[4], fabs(ida * aty));
    m[5] = fmax(m[5], fabs(ida * qa));
    m[10] = fmax(m[10], fabs(qa + aty));
    m[11] = fmax(m[11], fabs(aty));
    m[12] = fmax(m[12], fabs(qa));
  }
}
__device__ __forceinline__ void info_var_terms(const double dz, const double beta, const double x, const double zb,
                                               const double aty, const double px, const double qv, double (&m)[14]) {
  const double ax = beta * x;
  const double einv = dz / beta, dinv = 1.0 / dz;
  m[0] = fmax(m[0], fabs(einv * (ax - zb)));
  m[1] = fmax(m[1], fabs(einv * zb));
  m[2] = fmax(m[2], fabs(einv * ax));
  m[7] = fmax(m[7], fabs(ax - zb));
  m[8] = fmax(m[8], fabs(zb));
  m[9] = fmax(m[9], fabs(ax));
  const double d = qv + px + aty;
  m[3] = fmax(m[3], fabs(dinv * d));
  m[4] = fmax(m[4], fabs(dinv * aty));
  m[5] = fmax(m[5], fabs(dinv * qv));
  m[6] = fmax(m[6], fabs(dinv * px));
  m[10] = fmax(m[10], fabs(d));
  m[11] = fmax(m[11], fabs(aty));
  m[12] = fmax(m[12], fabs(qv));
  m[13] = fmax(m[13], fabs(px));
}
// first stage of the primal infeasibility certificate: a[0] |E dy| (max), a[1] u'dy+ + l'dy- (sum), a[2] |Dinv A_aux'dy|
// (max).  Returns the projected dual step of the row (the column pass of the second stage scatters it).
__device__ __forceinline__ double pinf_row_terms(const double* F, const int naux, double (&a)[3]) {
  double d = F[R_DY];
  d = (naux == AUX_HINGE) ? fmax(d, 0.0) : d;  // l = -inf
  a[0] = fmax(a[0], fabs(F[R_E] * d));
  a[1] += F[R_UP] * fmax(d, 0.0) + F[R_LO] * fmin(d, 0.0);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double da = fmin(F[R_DYA0 + k], 0.0);  // aux bound rows: u = +inf, l = 0
    a[0] = fmax(a[0], fabs(F[R_EA0 + k] * da));
    a[2] = fmax(a[2], fabs((F[R_U0 + k] * d + F[R_B0 + k] * da) / F[R_DA0 + k]));
  }
  return d;
}
__device__ __forceinline__ void pinf_var_terms(const double ratio, const double ub, const double lb, const double d,
                                               double (&a)[3]) {  // variable-bound rows: both bounds finite
  a[0] = fmax(a[0], fabs(ratio * d));
  a[1] += ub * fmax(d, 0.0) + lb * fmin(d, 0.0);
}
// first stage of the dual infeasibility certificate: a[0] |D dx| (max), a[1] q'dx (sum)
__device__ __forceinline__ void dinf_row_terms(const double* F, double (&a)[2]) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    a[0] = fmax(a[0], fabs(F[R_DA0 + k] * F[R_DXA0 + k]));
    a[1] += F[R_QA0 + k] * F[R_DXA0 + k];
  }
}
// Hash of the active-set guess the polish would start from (optimisation O1): an order-independent sum (mod 2^64) of
// one splitmix64 term per active row, keyed by the row's index in the canonical QP ([rows; trajectory bounds; aux
// bounds]) and the side it is active on.
__device__ __forceinline__ unsigned long long guess_mix(unsigned long long v) {
  v += 0x9e3779b97f4a7c15ull;
  v = (v ^ (v >> 30)) * 0xbf58476d1ce4e5b9ull;
  v = (v ^ (v >> 27)) * 0x94d049bb133111ebull;
  return v ^ (v >> 31);
}
__device__ __forceinline__ unsigned long long guess_row_hash(const double* F, const int* I, const int r, const int nrows,
                                                             const int N) {
  unsigned long long h = 0ull;
  const unsigned long long mc = static_cast<unsigned long long>(nrows);
  if (F[R_Z] - F[R_LO] < -F[R_Y]) h += guess_mix(2ull * r);
  else if (F[R_UP] - F[R_Z] < F[R_Y]) h += guess_mix(2ull * r + 1ull);
  for (int k = 0; k < I[RI_AUX]; ++k) {
    const unsigned long long idx = mc + N + I[RI_PAD] + k;
    if (F[R_ZA0 + k] - 0.0 < -F[R_YA0 + k]) h += guess_mix(2ull * idx);
    else if (kOsqpInf * F[R_EA0 + k] - F[R_ZA0 + k] < F[R_YA0 + k]) h += guess_mix(2ull * idx + 1ull);
  }
  return h;
}
__device__ __forceinline__ unsigned long long guess_var_hash(const double zb, const double yb, const double lb,
                                                             const double ub, const int i, const int nrows) {
  const unsigned long long idx = static_cast<unsigned long long>(nrows) + i;
  if (zb - lb < -yb) return guess_mix(2ull * idx);
  if (ub - zb < yb) return guess_mix(2ull * idx + 1ull);
  return 0ull;
}
// The check fused into admm_block_pinv leaves the warp partials of its quantities in the solver's Gauss-Jordan scratch
// (q.tmp, unused between factorisations): quantity k of warp w at [k * 8 + w], the guess hash as a 64-bit word at
// [kChkHash * 8 + w].  0..13 the norms of info_pass, then the first stages of the two certificates.
enum ChkQ { CHK_PA0 = 14, CHK_PA1, CHK_PA2, CHK_DA0, CHK_DA1, kChkHash };
constexpr unsigned kChkSumMask = (1u << CHK_PA1) | (1u << CHK_DA1);

// per-row weights of the current linear system -> R_WRR (raw row weight), R_G0/G1, R_DEN, R_WR (Schur weight).
// With the aux block K_aa = diag(g) + Wr u u' everything is written cancellation free (den = det K_aa
// expanded analytically); the polish system has Wr = 1/delta and g = delta.
__device__ inline void rows_prepare_weights(const QpCtx& q, const SysW& w) {
  for (int r = q.tid; r < q.nrows; r += kQpThreads) {
    double* F = q.F(r);
    const int naux = q.I(r)[RI_AUX];
    const double Wr = w.polish ? fabs(F[R_PW]) : ((F[R_RHO] != 0.0) ? q.rho_eq : q.rho);
    const double wa0 = w.polish ? fabs(F[R_PWA0]) : w.rho_aux;
    const double wa1 = w.polish ? fabs(F[R_PWA1]) : w.rho_aux;
    const double g0 = (naux >= 1) ? w.sig + wa0 * F[R_B0] * F[R_B0] : 1.0;
    const double g1 = (naux == 2) ? w.sig + wa1 * F[R_B1] * F[R_B1] : 1.0;
    const double den = g0 * g1 + Wr * (F[R_U0] * F[R_U0] * g1 + F[R_U1] * F[R_U1] * g0);
    F[R_WRR] = Wr;
    F[R_G0] = g0;
    F[R_G1] = g1;
    F[R_DEN] = den;
    F[R_IDEN] = 1.0 / den;
    F[R_IWRR] = (Wr != 0.0) ? 1.0 / Wr : 0.0;
    F[R_WR] = Wr * g0 * g1 / den;
  }
  __syncthreads();
}
__device__ __forceinline__ double xbound_weight(const QpCtx& q, const SysW& w, int j) {
  const double adm = (q.ubs[j] - q.lbs[j] < kRhoTol) ? q.rho_eq : q.rho;
  return w.polish ? fabs(q.zb[j]) : adm;  // zb holds the signed polish weights during polish
}

// K = P + sig I + A' W A with the aux variables eliminated, written straight into the block storage
// (SA: diagonal blocks, SLM: left couplings); one thread per matrix row; then factor.
// ---- partition-inverse factorisation (PinvPlan) -----------------------------------------------------------------------
// In-place Gauss-Jordan inverse of independent SPD matrices, one thread per row with the row in registers (a[QN],
// zeros beyond the matrix size n).  Register arrays cannot be indexed by the (run-time) step number, and unrolling the
// steps (6 k instructions) ran at the speed of the instruction fetch, rotating the row (2 QN register moves per step)
// at the speed of instruction issue, and anything the pivot thread does to its own row sits on the critical path of the
// step (its warp runs both sides of the branch).  So the columns stay put, every step is the same generic update
// a[j] -= g' t[j] over ALL columns with compile-time indices, and what depends on the step is carried as scales:
//  * the thread's entry f of the pivot column comes from the published pivot row: the working matrix is symmetric in
//    the rows still to be eliminated and antisymmetric across the eliminated ones;
//  * the finished column k (true value -f / pivot in the other rows) is not written: the pivot thread publishes 0 in
//    place of its pivot entry, the column keeps f and carries the scale -1 / pivot from then on (one per column and
//    matrix, in shared memory);
//  * the pivot row is not scaled either: it carries the row scale 1 / pivot (a register), and its later updates use
//    g / scale = g * pivot;
//  * the diagonal entry of an eliminated row does not fit either scale: it lives in a register of its own (as the
//    not-yet-eliminated rows' diagonal entries do, together with their reciprocal, ready for the row's own pivot step).
// One pass at the end applies the scales.  scripts/probes/pinv_proto.py holds the same algorithm in numpy (error 1e-15
// at condition 1e16; a shortcut that published pivot + 1 to get -g by cancellation lost eps * pivot).
// tmp: [2][nmat][QN + 2] then [nmat][QN] column scales.  Called by the 64 threads of the two warps that hold every row
// of matrix `mat`: one named barrier (`bar.sync bar, 64`) per step, n_max steps.  (Named barriers 1 and 2 also serve
// eval_step, which a CTA never runs while it is in a QP step: solve_kernel separates the two by CTA barriers.)  Returns
// true when this thread met a non-positive pivot.
// 1 / x for the pivots: hardware seed (about 20 bits) and three Newton steps, straight-line code (the library division
// keeps a slow-path CALL, and a call inside the elimination loop spills the row around it)
__device__ __forceinline__ double pivot_rcp(const double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  return fma(r, e, r);
}
template <int QN>
__device__ __forceinline__ bool gj_rows(double (&a)[QN], double diag, const bool active, const int mat, const int row,
                                        const int n, const int n_max, double* tmp, const int nmat, const int bar) {
  constexpr int BS = QN + 2;  // row + reciprocal (+ pad)
  double* const csv = tmp + 2 * nmat * BS + mat * QN;  // this matrix's column scales
  bool bad = false;
  // diag: the row's diagonal entry (true value; after the row's own step: of the inverse being built)
  double pv_mine = pivot_rcp(diag), my_cs = 1.0, rs = 1.0, inv_rs = 1.0;
#pragma unroll 1
  for (int k = 0; k < n_max; ++k) {
    double* buf = tmp + ((k & 1) * nmat + mat) * BS;
    const bool piv = active && row == k;  // (k < n follows from row < n)
    if (piv) {
      bad |= !(diag > 0.0);
#pragma unroll
      for (int j = 0; j < QN; j += 2) *reinterpret_cast<double2*>(buf + j) = make_double2(a[j], a[j + 1]);
      buf[k] = 0.0;
      buf[QN] = pv_mine;
      my_cs = -pv_mine;
      csv[k] = my_cs;
      rs = pv_mine;
      inv_rs = diag;
      diag = pv_mine;
    }
    asm volatile("bar.sync %0, 64;" ::"r"(bar) : "memory");
    if (active && k < n && !piv) {
      const double tr = buf[row];
      const bool ahead = row > k;  // this row is still to be eliminated
      const double f = ahead ? tr : -tr * my_cs;
      const double g = f * buf[QN];
      diag = ahead ? diag - g * f : diag + g * f;
      const double gs = g * inv_rs;
#pragma unroll
      for (int j = 0; j < QN; j += 2) {
        const double2 t = *reinterpret_cast<const double2*>(buf + j);
        a[j] -= gs * t.x;
        a[j + 1] -= gs * t.y;
      }
      if (ahead) pv_mine = pivot_rcp(diag);
    }
  }
  if (active) {
#pragma unroll
    for (int j = 0; j < QN; ++j) a[j] = (j == row) ? diag : ((j < n) ? a[j] * (rs * csv[j]) : 0.0);
  }
  return bad;
}

// From the assembled blocks (SA: diagonal blocks, SLM: K(block p, block p-1)) to PI (global, read back into registers
// by admm_block_pinv), W, Z (shared).  Called by every thread of the CTA.  false: a pivot was not positive.
template <int NB>
__device__ inline bool pinv_factor(const QpCtx& q) {
  constexpr int QN = 3 * NB, blk = NB * NB;
  static_assert(QN % 2 == 0, "pivot rows move as double2");
  static_assert(QN <= 64, "a partition on two warps");
  extern __shared__ double sm[];
  const int tid = q.tid, M = q.M, Np = q.Np;
  const int PR = q.pl.PR, nS = q.pl.nS, Ns = q.pl.Ns, ZS = q.pl.ZS, WS = q.pl.WS, SS = q.pl.SS;
  double* const fbase = sm + (q.SA - q.smbase);
  const double* const SA = fbase;
  const double* const SLM = sm + (q.SLM - q.smbase);
  double* const Z = fbase + q.pl.zo;
  double* const W = fbase + q.pl.wo;
  double* const S = fbase + q.pl.so;
  double* const tmp = q.tmp.ptr();
  const int nparts = (M + 3) / 4;
  bool bad = false;
#ifdef TB200_PROFILE
  long long pf_ = clock64();
#define PROF_PF(slot) do { const long long n_ = clock64(); if (tid == 0) atomicAdd(&g_prof[slot], (unsigned long long)(n_ - pf_)); pf_ = n_; } while (0)
#else
#define PROF_PF(slot)
#endif
  {
    // ---- 1. inverse of every partition (the tridiagonal run of <= 3 blocks starting at block 4 p): partition p on warps
    // 2p and 2p + 1, its rows on their first lanes; row lr of partition p is row pr = p QN + lr of PI and W
    const int p = tid >> 6, lr = tid & 63, pr = p * QN + lr;
    const bool part = p < nparts;
    const int npb = !part ? 0 : (M - 4 * p) < 3 ? (M - 4 * p) : 3;
    const bool prow = lr < npb * NB;
    const int kb = lr / NB, r = lr % NB, gb = 4 * p + kb;  // local block, row inside it, global block
    double a[QN];
#pragma unroll
    for (int j = 0; j < QN; ++j) {
      const int cb = j / NB, c = j % NB;  // (compile-time)
      double v = 0.0;
      if (prow && cb < npb) {
        if (cb == kb) v = SA[gb * blk + r * NB + c];
        else if (cb == kb - 1) v = SLM[gb * blk + r * NB + c];            // K(gb, gb - 1)
        else if (cb == kb + 1) v = SLM[(gb + 1) * blk + c * NB + r];      // K(gb, gb + 1) = K(gb + 1, gb)'
      }
      a[j] = v;
    }
    PROF_PF(0);
    const double dg = prow ? SA[gb * blk + r * NB + r] : 1.0;  // the row's diagonal entry
    if (part) bad |= gj_rows<QN>(a, dg, prow, p, lr, npb * NB, (M < 3 ? M : 3) * NB, tmp, nparts, 1 + p);
    PROF_PF(4);
    if (prow) {
#pragma unroll
      for (int j = 0; j < QN; ++j) q.pi_g[j * PR + pr] = a[j];
      // ---- 2. W = PI C: the left separator couples to the partition's first block (C = SLM[4p]), the right one to its
      // last block (C = SLM[4p + 3]'); a partition that has a right separator is always full (3 blocks)
      const bool has_l = p > 0, has_r = 4 * p + 3 < M;
#pragma unroll 2
      for (int j = 0; j < NB; ++j) {
        double wl = 0.0, wr = 0.0;
        if (has_l) {
#pragma unroll
          for (int c = 0; c < NB; ++c) wl += a[c] * SLM[(4 * p) * blk + c * NB + j];
        }
        if (has_r) {
#pragma unroll
          for (int c = 0; c < NB; ++c) wr += a[2 * NB + c] * SLM[(4 * p + 3) * blk + j * NB + c];
        }
        W[pr * WS + j] = wl;
        W[pr * WS + NB + j] = wr;
      }
    }
  }
  __syncthreads();
  // ---- 3. Schur complement on the separators: S = A_ss - C' W (block tridiagonal in the separators).  One entry per
  // thread and pass; the dot products are unrolled with two partial sums each (a single dependent chain of 28
  // multiply-adds with its loads in between is bound by their latency)
  for (int e = tid; e < nS * nS; e += kQpThreads) {
    const int ra = e / nS, ca = e % nS, sa = ra / NB, i = ra % NB, sb = ca / NB, j = ca % NB;
    double v = 0.0;
    if (sa == sb || sb == sa + 1 || sb == sa - 1) {
      // left partition of separator sa (its last block couples through SLM[4 sa + 3](i, :)), right partition (its first
      // block couples through SLM[4 sa + 4](:, i)); the W columns: the partition's own left (0) or right (NB) separator
      const bool use_l = sb <= sa, use_r = sb >= sa && 4 * sa + 4 < M;
      const double* cl = SLM + (4 * sa + 3) * blk + i * NB;                       // stride 1 over rr
      const double* wl = W + (sa * QN + 2 * NB) * WS + (sb == sa ? NB : 0) + j;   // stride WS over rr
      const double* cr = SLM + (4 * sa + 4) * blk + i;                            // stride NB over rr
      const double* wr = W + ((sa + 1) * QN) * WS + (sb == sa ? 0 : NB) + j;      // stride WS over rr
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      if (use_l) {
#pragma unroll
        for (int rr = 0; rr < NB; rr += 2) {
          s0 += cl[rr] * wl[rr * WS];
          s1 += cl[rr + 1] * wl[(rr + 1) * WS];
        }
      }
      if (use_r) {
#pragma unroll
        for (int rr = 0; rr < NB; rr += 2) {
          s2 += cr[rr * NB] * wr[rr * WS];
          s3 += cr[(rr + 1) * NB] * wr[(rr + 1) * WS];
        }
      }
      v = ((sa == sb) ? SA[(4 * sa + 3) * blk + i * NB + j] : 0.0) - ((s0 + s1) + (s2 + s3));
    }
    S[ra * SS + ca] = v;
  }
  __syncthreads();
  PROF_PF(14);
  {
    // ---- 4. its inverse (one matrix of nS <= 3 NB rows)
    const bool srow = tid < nS;
    double a[QN];
#pragma unroll
    for (int j = 0; j < QN; ++j) a[j] = (srow && j < nS) ? S[tid * SS + j] : 0.0;
    const double dg = srow ? S[tid * SS + tid] : 1.0;
    if (tid < 64) bad |= gj_rows<QN>(a, dg, srow, 0, tid, nS, nS, tmp, 1, 1);  // (nS <= 3 NB rows: warps 0 and 1)
    if (srow) {
#pragma unroll
      for (int j = 0; j < QN; ++j)
        if (j < nS) S[tid * SS + j] = a[j];
    }
  }
  __syncthreads();
  PROF_PF(15);
  // ---- 5. Z = [-Sinv W' | Sinv]: the separator rows of the inverse of the whole matrix (over the dead SA / SLM).
  // One thread per COLUMN with its row of W in registers; per separator row 2 NB multiply-adds against a row segment of
  // Sinv that every thread of the partition reads at the same address; the stores of a warp are contiguous.
  if (tid < Np) {
    const int col = tid, cb = col / NB, c = col % NB, p = cb / 4;
    if (cb % 4 == 3) {
      for (int sr = 0; sr < nS; ++sr) Z[sr * ZS + col] = S[sr * SS + p * NB + c];
    } else {
      const bool has_l = p > 0, has_r = 4 * p + 3 < M;
      const double* wrow = W + (p * QN + (cb % 4) * NB + c) * WS;
      double wv[2 * NB];
#pragma unroll
      for (int t = 0; t < 2 * NB; ++t) wv[t] = wrow[t];
      const double* sl = S + (has_l ? (p - 1) * NB : 0);  // (W is zero where a separator is absent)
      const double* sr_ = S + (has_r ? p * NB : 0);
#pragma unroll 2
      for (int sr = 0; sr < nS; ++sr) {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
        for (int t = 0; t < NB; t += 2) {
          s0 += sl[sr * SS + t] * wv[t];
          s1 += sl[sr * SS + t + 1] * wv[t + 1];
          s2 += sr_[sr * SS + t] * wv[NB + t];
          s3 += sr_[sr * SS + t + 1] * wv[NB + t + 1];
        }
        Z[sr * ZS + col] = -((s0 + s1) + (s2 + s3));
      }
    }
  }
  (void)Ns;
  const bool ok = !__syncthreads_or(bad ? 1 : 0);
  PROF_PF(9);
  return ok;
}

// PINV: the partition-inverse form (pinv_factor), else the cyclic reduction (bcr_factor<NB, WARP>)
template <int NB, bool PINV, bool WARP>
__device__ __noinline__ bool assemble_factor(const QpCtx& q, const SysW& w) {
  PROF_T0();
  rows_prepare_weights(q, w);
  constexpr int nb = NB, blk = NB * NB;
  // (both forms that run on chip address the factor as shared memory; the global-memory factor and the CTA-wide
  // reference keep generic pointers)
  extern __shared__ double sm[];
  constexpr bool SMEM = PINV || WARP;
  double* const SA = SMEM ? sm + (q.SA - q.smbase) : q.SA;
  double* const SLM = SMEM ? sm + (q.SLM - q.smbase) : q.SLM;
  const int N = q.N, HB = 2 * q.D, PW = HB + 1, CN = q.CN;
  for (int t = q.tid; t < q.M * blk; t += kQpThreads) {
    SA[t] = 0.0;
    SLM[t] = 0.0;
  }
  __syncthreads();
  for (int i = q.tid; i < q.Np; i += kQpThreads) {
    const int p = i / nb, r = i % nb;
    double* Arow = SA + static_cast<size_t>(p) * blk + r * nb;   // K(i, p*nb + c)
    double* Lrow = SLM + static_cast<size_t>(p) * blk + r * nb;   // K(i, (p-1)*nb + c)
    if (i >= N) {
      Arow[r] = 1.0;  // padding variable
      continue;
    }
    // element K(i, i-k), k = 0..HB, lands in the diagonal block (k <= r) or the left coupling block.  (__dadd_rn: the
    // sum is never contracted with the product that forms val, whatever the addressing lets the compiler schedule, so
    // that every factor form assembles the same bits)
    auto add = [&](int k, double val) {
      if (k <= r) Arow[r - k] = __dadd_rn(Arow[r - k], val);
      else Lrow[nb + r - k] = __dadd_rn(Lrow[nb + r - k], val);
    };
    for (int t = 0; t < q.n_band; ++t) {
      const int k = q.band_offs[t];
      if (k <= i) add(k, q.c * q.Dz[i] * q.Pband[i * PW + k] * q.Dz[i - k]);
    }
    add(0, w.sig + xbound_weight(q, w, i) * q.beta[i] * q.beta[i]);
    for (int e = q.colptr[i]; e < q.colptr[i + 1]; ++e) {
      const int ent = q.colent[e], rw = ent >> 5, k = ent & 31;
      const double* R = q.R(rw);
      const double wr = R[2 * CN + R_WR];
      if (wr == 0.0) continue;
      const int stride = q.I(rw)[RI_STRIDE];
      const double* as = R + CN;
      const double ai = wr * as[k];
      for (int k2 = 0; k2 <= k; ++k2) add((k - k2) * stride, ai * as[k2]);
    }
  }
  __syncthreads();
  // mirror the strictly lower part of every diagonal block into its upper part
  for (int t = q.tid; t < q.M * blk; t += kQpThreads) {
    const int p = t / blk, i = (t % blk) / nb, j = t % nb;
    if (j > i) SA[static_cast<size_t>(p) * blk + i * nb + j] = SA[static_cast<size_t>(p) * blk + j * nb + i];
  }
  __syncthreads();
  // slots 24 + 2 kind (assembly) and 25 + 2 kind (elimination); kind: 0 initial, 1 rho update or recovery, 2 polish
#ifdef TB200_PROFILE
  const int pk = w.polish ? 2 : w.prof_kind;
  if (pk == 1) PROF_COUNT(31);
#endif
  PROF_ADD2(10, 24 + 2 * pk);
  bool ok;
  {
    PROF_T0();
    if constexpr (PINV) ok = pinv_factor<NB>(q);
    else ok = bcr_factor<NB, WARP>(q);
    PROF_ADD2(11, 25 + 2 * pk);
  }
  return ok;
}

// The code paths of one QP solve (qp_solve_block), decided by the layout of the QP:
//   use_reg:     the ADMM loop keeps the thread's rows of the factor in registers when the roles fit the CTA
//   use_pinv:    short trajectories with their rows on chip use the partition-inverse form of the system (PinvPlan)
//   fuse:        the partition-inverse block can end in the terms of a termination check ...
//   fast_polish: ... and the polish refinement runs as polish_passes (else the generic passes of qp_solve_block)
// regok: the register-resident solve may be used (blocks of <= 14); fast_passes: DevProblem::qp_fast_passes.
struct QpPlan {
  bool use_reg, use_pinv, fuse, fast_polish;
};
__host__ __device__ inline QpPlan qp_plan(bool regok, int pinv, int rows_smem, int M, int nb, bool fast_passes) {
  QpPlan pl;
  pl.use_reg = regok && solve_roles_fit(M, nb);
  pl.use_pinv = regok && pinv && rows_smem;
  pl.fuse = pl.use_pinv && fast_passes;
  pl.fast_polish = pl.use_pinv && fast_passes && M * nb <= kQpThreads && solve_roles_fit(M, nb);
  return pl;
}
// The code paths of a QP as bits (tb200_debug_qp_paths: ORed per trajectory over its QPs when recording is on)
enum QpPath {
  QPP_BLOCK_PINV = 1 << 0,      // ADMM blocks: admm_block_pinv
  QPP_BLOCK_FAST = 1 << 1,      //              admm_block_fast
  QPP_BLOCK_GENERIC = 1 << 2,   //              admm_block
  QPP_BLOCK_SOA = 1 << 3,       //              admm_block_soa (rows in global memory)
  QPP_FACTOR_GLOBAL = 1 << 4,   // the factor in this CTA's region of global memory
  QPP_BAND_GLOBAL = 1 << 5,     // the objective band read from global memory
  QPP_ROWS_GLOBAL = 1 << 6,     // the rows of the QP in global memory (more than row_cap)
  QPP_FUSED_CHECK = 1 << 7,     // the termination checks take the residuals fused into admm_block_pinv
  QPP_POLISH_FAST = 1 << 8,     // a polish was refined through polish_passes
  QPP_POLISH_GENERIC = 1 << 9   // a polish was refined through the generic passes
};
// the ADMM block a plan runs (the choice of qp_solve_block's run_block)
__host__ __device__ inline int qp_plan_block(const QpPlan& pl, int rows_smem) {
  if (pl.use_pinv) return QPP_BLOCK_PINV;
  if (!rows_smem) return QPP_BLOCK_SOA;
  return pl.use_reg ? QPP_BLOCK_FAST : QPP_BLOCK_GENERIC;
}

struct QpOut {
  int status, iters, polish;
  double rho;
  double pri_res, dua_res, pol_pri, pol_dua, c;
  int pol_factor_ok, rho_updates, rounds;
};

// Scatter pass: v1[i] = base(i) + sum over the column entries of as[k] * R_COEF(row).
template <int CN, class Base>
__device__ __forceinline__ void scatter_columns(const QpCtx& q, Base base) {
  for (int i = q.tid; i < q.Np; i += kQpThreads) {
    double s = 0.0;
    if (i < q.N) {
      s = base(i);
      for (int e = q.colptr[i]; e < q.colptr[i + 1]; ++e) {
        const int ent = q.colent[e], r = ent >> 5, k = ent & 31;
        const double* R = q.R(r);
        s += R[CN + k] * R[2 * CN + R_COEF];
      }
    }
    q.v1[i] = s;
  }
  __syncthreads();
}
// zeta_r = as . v(vars of the row); all CN (zero padded) coefficients
template <int CN>
__device__ __forceinline__ double row_dot(const QpCtx& q, const double* R, const int* I, const double* v) {
  double z = 0.0;
  const int base = I[RI_BASE], stride = I[RI_STRIDE], last = I[RI_CNT] - 1;
#pragma unroll
  for (int k = 0; k < CN; ++k) z += R[CN + k] * v[base + min(k, last) * stride];
  return z;
}
// aux back-substitution (cancellation free; absent aux slots have u = ra = 0 and g = 1 and come out 0)
__device__ __forceinline__ void row_backsub(const double* F, double zeta, double& a0, double& a1) {
  const double Wr = F[R_WRR], ra0 = F[R_RA0], ra1 = F[R_RA1], u0 = F[R_U0], u1 = F[R_U1];
  const double iden = F[R_IDEN];
  a0 = (F[R_G1] * (ra0 - Wr * u0 * zeta) + Wr * u1 * (u1 * ra0 - u0 * ra1)) * iden;
  a1 = (F[R_G0] * (ra1 - Wr * u1 * zeta) + Wr * u0 * (u0 * ra1 - u1 * ra0)) * iden;
}
__device__ __forceinline__ double row_reduce_coef(const double* F, double ra0, double ra1, double zcoef) {
  return zcoef - F[R_WRR] * (F[R_U0] * ra0 * F[R_G1] + F[R_U1] * ra1 * F[R_G0]) * F[R_IDEN];
}
// The row work of the ADMM blocks whose rows are records (R, F, I): admm_block passes q.R(r), q.F(r), q.I(r), the
// others their shared-memory offsets.  The scalars are references so that admm_block, which passes the fields of its
// context, reads them where they are used (copies held across the row's stores cost it spills); the others pass
// locals.  Entry pass: the aux right-hand sides R_RA0/1, the row multiplier R_COEF and the row's contributions to the
// right-hand side of the next solve, from the current row state.
template <int CNc>
__device__ __forceinline__ void admm_row_entry(const double* R, double* F, const double& sigma, const double& rho_aux) {
  const double s = F[R_WRR] * F[R_Z] - F[R_Y];
  const double ra0 = sigma * F[R_XA0] - F[R_QA0] + F[R_U0] * s + F[R_B0] * (rho_aux * F[R_ZA0] - F[R_YA0]);
  const double ra1 = sigma * F[R_XA1] - F[R_QA1] + F[R_U1] * s + F[R_B1] * (rho_aux * F[R_ZA1] - F[R_YA1]);
  F[R_RA0] = ra0;
  F[R_RA1] = ra1;
  const double cf = row_reduce_coef(F, ra0, ra1, s);
  F[R_COEF] = cf;
#pragma unroll
  for (int k = 0; k < CNc; ++k) F[R_NF + k] = R[CNc + k] * cf;
}
// After a solve w: back-substitute aux, relax, project, dual update, and the multipliers for the next solve
// (oma = 1 - alpha, inv_rho_aux = 1 / rho_aux).
template <int CNc>
__device__ __forceinline__ void admm_row_update(const double* R, double* F, const int* I, const double* w,
                                                const double& sigma, const double& alpha, const double& oma,
                                                const double& rho_aux, const double& inv_rho_aux) {
  double zeta = 0.0;
  {
    const int base = I[RI_BASE], stride = I[RI_STRIDE], last = I[RI_CNT] - 1;
#pragma unroll
    for (int k = 0; k < CNc; ++k) zeta += R[CNc + k] * w[base + min(k, last) * stride];
  }
  double a0, a1;
  row_backsub(F, zeta, a0, a1);
  const double zt = zeta + F[R_U0] * a0 + F[R_U1] * a1;
  const double Wr = F[R_WRR];
  const double zr = alpha * zt + oma * F[R_Z];
  double zn = zr + F[R_Y] * F[R_IWRR];
  zn = fmin(fmax(zn, F[R_LO]), F[R_UP]);
  const double dy = Wr * (zr - zn);
  const double yn = F[R_Y] + dy;
  F[R_Z] = zn;
  F[R_Y] = yn;
  F[R_DY] = dy;
  const double s = Wr * zn - yn;
  double ra[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double at = k ? a1 : a0, bb = F[R_B0 + k];
    const double xo = F[R_XA0 + k];
    const double xn = alpha * at + oma * xo;
    const double zra = alpha * (bb * at) + oma * F[R_ZA0 + k];
    double z2 = zra + F[R_YA0 + k] * inv_rho_aux;
    z2 = fmin(fmax(z2, 0.0), kOsqpInf * F[R_EA0 + k]);
    const double dya = rho_aux * (zra - z2);
    const double yan = F[R_YA0 + k] + dya;
    F[R_XA0 + k] = xn;
    F[R_DXA0 + k] = xn - xo;
    F[R_ZA0 + k] = z2;
    F[R_YA0 + k] = yan;
    F[R_DYA0 + k] = dya;
    ra[k] = sigma * xn - F[R_QA0 + k] + F[R_U0 + k] * s + bb * (rho_aux * z2 - yan);
  }
  F[R_RA0] = ra[0];
  F[R_RA1] = ra[1];
  const double cf = row_reduce_coef(F, ra[0], ra[1], s);
  F[R_COEF] = cf;
#pragma unroll
  for (int k = 0; k < CNc; ++k) F[R_NF + k] = R[CNc + k] * cf;
}

// ---------------------------------------------------------------------------------------------------
// A block of ADMM iterations (no termination test inside): its own function (not inlined), so that the loop the
// whole batch time hangs on has its own register allocation and sits in one contiguous piece of code — the rest of
// the solver (scaling, residuals, certificates, polish, factorisation) cannot spill into it or push it out of the
// instruction cache.  The generic solve reads the factor rows from memory.  Rows are handled by the high thread ids
// so that they run beside the per-variable work of the low ones.  Every iteration leaves the aux right-hand sides
// R_RA0/1, the row multiplier R_COEF and the rows' contributions to the right-hand side of the next solve behind; the
// entry pass (re)builds them because the residual passes, the polish and a refactorisation reuse those fields.
// keep_last: the last iteration records its primal / dual steps (dxs, dyb) for the infeasibility certificates.
template <int NB, int PAIR>
__device__ __noinline__ void admm_block(const QpCtx& q, const double rho_aux, const int n_iter, const int keep_last) {
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  const int N = q.N, tid = q.tid;
  double* const dxs = q.scratch;
  double* const dyb = q.scratch + q.Np;
  const bool one_var = q.Np <= kQpThreads;  // one thread per variable: its column range is loop invariant
  const int my_e0 = (one_var && tid < N) ? q.colptr[tid] : 0, my_e1 = (one_var && tid < N) ? q.colptr[tid + 1] : 0;
  {  // entry pass: aux right-hand sides, row multipliers and contributions from the current row state
    PROF_T0();
    for (int r = kQpThreads - 1 - tid; r < q.nrows; r += kQpThreads)
      admm_row_entry<CNc>(q.R(r), q.F(r), q.sigma, rho_aux);
    __syncthreads();
    PROF_ADD(0);
  }
  const double inv_rho_aux = 1.0 / rho_aux;
  const double inv_rho = 1.0 / q.rho, inv_rho_eq = 1.0 / q.rho_eq;
  for (int it = 0; it < n_iter; ++it) {
    const bool keep_steps = keep_last && it == n_iter - 1;
    // right-hand side  sigma x - q + A'(rho z - y)  (one thread per variable; the rows left their terms behind)
    {
      PROF_T0();
      if (one_var) {
        const int i = tid;
        double s = 0.0;
        if (i < N) {
          const double rb = (q.ubs[i] - q.lbs[i] < kRhoTol) ? q.rho_eq : q.rho;
          s = q.sigma * q.x[i] - q.qs[i] + q.beta[i] * (rb * q.zb[i] - q.yb[i]);
          for (int e = my_e0; e < my_e1; ++e) {
            const int ent = q.colent[e];
            s += q.rows[static_cast<size_t>(ent >> 5) * q.RS + (2 * CNc + R_NF) + (ent & 31)];
          }
        }
        if (i < q.Np) q.v1[i] = s;
      } else {
        for (int i = tid; i < q.Np; i += kQpThreads) {
          double s = 0.0;
          if (i < N) {
            const double rb = (q.ubs[i] - q.lbs[i] < kRhoTol) ? q.rho_eq : q.rho;
            s = q.sigma * q.x[i] - q.qs[i] + q.beta[i] * (rb * q.zb[i] - q.yb[i]);
            for (int e = q.colptr[i]; e < q.colptr[i + 1]; ++e) {
              const int ent = q.colent[e];
              s += q.rows[static_cast<size_t>(ent >> 5) * q.RS + (2 * CNc + R_NF) + (ent & 31)];
            }
          }
          q.v1[i] = s;
        }
      }
      PROF_ADD(1);
    }
    {
      PROF_T0();
      bcr_solve<NB>(q, q.v1, q.w);
      PROF_ADD(2);
    }
    PROF_T0();
    // rows: back-substitute aux, relax, project, dual update, and the multipliers for the next solve
    for (int r = kQpThreads - 1 - tid; r < q.nrows; r += kQpThreads)
      admm_row_update<CNc>(q.R(r), q.F(r), q.I(r), q.w, q.sigma, q.alpha, 1.0 - q.alpha, rho_aux, inv_rho_aux);
    // trajectory variables and their bound rows (one thread per variable)
    for (int i = tid; i < N; i += kQpThreads) {
      const double beta = q.beta[i];
      const double lb = q.lbs[i], ub = q.ubs[i];
      const bool beq = ub - lb < kRhoTol;
      const double rb = beq ? q.rho_eq : q.rho, irb = beq ? inv_rho_eq : inv_rho;
      const double xt = q.w[i];
      const double xn = q.alpha * xt + (1.0 - q.alpha) * q.x[i];
      const double zr = q.alpha * (beta * xt) + (1.0 - q.alpha) * q.zb[i];
      double zn = zr + q.yb[i] * irb;
      zn = fmin(fmax(zn, lb), ub);
      const double dy = rb * (zr - zn);
      if (keep_steps) {
        dxs[i] = xn - q.x[i];
        dyb[i] = dy;
      }
      q.x[i] = xn;
      q.zb[i] = zn;
      q.yb[i] += dy;
    }
    __syncthreads();
    PROF_ADD(3);
  }
}

// The same block of iterations for the common case — the solve's thread roles fit the CTA, QP rows in shared
// memory — written for the latency of ONE iteration:
//  * every operand address is an offset into the CTA's dynamic shared memory (LDS / STS, not generic loads), every
//    solver scalar a register (the QpCtx behind `q` is only read at entry);
//  * the thread's variable (x, z, y of its bound row, its scaling, bounds, cost) lives in registers for the whole block
//    and goes back to shared memory at the end: the right-hand side of the next solve is built from registers plus the
//    rows' contributions, which are fetched through entry addresses preloaded once per block (8 per variable, the
//    common case; longer columns walk the rest of their list);
//  * nothing loop invariant is recomputed inside the loop.
// The row work is admm_block's (admm_row_entry, admm_row_update); the variable's update keeps its operations and
// their order.
template <int NB, int PAIR>
__device__ __noinline__ void admm_block_fast(const QpCtx& q, const double rho_aux_in, const int n_iter, const int keep_last) {
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  constexpr int kPre = 8;  // column entries whose addresses are kept in registers
  extern __shared__ double sm[];
  const int tid = q.tid, N = q.N, Np = q.Np, nrows = q.nrows, RS = q.RS;
  const double sigma = q.sigma, alpha = q.alpha, oma = 1.0 - q.alpha, rho = q.rho, rho_eq = q.rho_eq, rho_aux = rho_aux_in;
  const double inv_rho_aux = 1.0 / rho_aux, inv_rho = 1.0 / rho, inv_rho_eq = 1.0 / rho_eq;
  double* const v1 = sm + (q.v1 - q.smbase);
  double* const w = sm + (q.w - q.smbase);
  double* const rows = sm + (q.rows - q.smbase);
  const int* const rints = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.rints) - q.smbase));
  const int* const colent = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.colent) - q.smbase));
  double* const dxs = q.scratch;
  double* const dyb = q.scratch + Np;
  const SolveRoles roles = solve_roles<NB>(q);
  double mB0[NB + NB / 2];  // the thread's level-0 backward row of the factor
  load_bwd_row<NB>(q, 0, tid, mB0);
  // ---- this thread's variable
  const bool has_var = tid < N;
  const int vi = has_var ? tid : 0;
  const double v_beta = q.beta[vi], v_lb = q.lbs[vi], v_ub = q.ubs[vi], v_qs = q.qs[vi];
  const bool v_eq = v_ub - v_lb < kRhoTol;
  const double v_rb = v_eq ? rho_eq : rho, v_irb = v_eq ? inv_rho_eq : inv_rho;
  double v_x = q.x[vi], v_z = q.zb[vi], v_y = q.yb[vi];
  const int e0 = has_var ? q.colptr[vi] : 0, e1 = has_var ? q.colptr[vi + 1] : 0;
  // a word that always reads 0.0: the padding coefficient of row 0's contribution block does not exist, so the zero
  // comes from the (unused) last scalar slot of the factorisation scratch
  double* const zero_slot = sm + (q.flag - q.smbase) + 7;
  if (tid == 0) *zero_slot = 0.0;
  int ea[kPre];
#pragma unroll
  for (int k = 0; k < kPre; ++k) {
    const int e = e0 + k;
    const int ent = (e < e1) ? colent[e] : -1;
    ea[k] = (ent >= 0) ? static_cast<int>(rows - sm) + (ent >> 5) * RS + (2 * CNc + R_NF) + (ent & 31)
                       : static_cast<int>(zero_slot - sm);
  }
  // ---- this thread's row (rows are handled by the high thread ids so that they run beside the per-variable work)
  {  // entry pass: aux right-hand sides, row multipliers and contributions from the current row state
    PROF_T0();
    for (int r = kQpThreads - 1 - tid; r < nrows; r += kQpThreads)
      admm_row_entry<CNc>(rows + r * RS, rows + r * RS + 2 * CNc, sigma, rho_aux);
    __syncthreads();
    PROF_ADD(0);
  }
  for (int it = 0; it < n_iter; ++it) {
    const bool keep_steps = keep_last && it == n_iter - 1;
    {
      PROF_T0();
      // right-hand side  sigma x - q + A'(rho z - y): the variable's own part from registers, the rows left their terms behind
      double s = 0.0;
      if (has_var) {
        s = sigma * v_x - v_qs + v_beta * (v_rb * v_z - v_y);
        double c[kPre];
#pragma unroll
        for (int k = 0; k < kPre; ++k) c[k] = sm[ea[k]];
        // (a fixed pairwise order: the eight loads are in flight together instead of one load per dependent add)
        if constexpr (kPre == 8) s += ((c[0] + c[1]) + (c[2] + c[3])) + ((c[4] + c[5]) + (c[6] + c[7]));
        else s += (c[0] + c[1]) + (c[2] + c[3]);
        for (int e = e0 + kPre; e < e1; ++e) {
          const int ent = colent[e];
          s += rows[(ent >> 5) * RS + (2 * CNc + R_NF) + (ent & 31)];
        }
      }
      if (tid < Np) v1[tid] = s;
      PROF_ADD(1);
    }
    {
      PROF_T0();
      bcr_solve_hyb<NB>(tid, roles, mB0, sm, v1, w);
      PROF_ADD(2);
    }
    PROF_T0();
    // rows: back-substitute aux, relax, project, dual update, and the multipliers for the next solve
    for (int r = kQpThreads - 1 - tid; r < nrows; r += kQpThreads)
      admm_row_update<CNc>(rows + r * RS, rows + r * RS + 2 * CNc, rints + r * RI_NINTS, w, sigma, alpha, oma, rho_aux,
                           inv_rho_aux);
    // the thread's variable and its bound row
    if (has_var) {
      const double xt = w[vi];
      const double xn = alpha * xt + oma * v_x;
      const double zr = alpha * (v_beta * xt) + oma * v_z;
      double zn = zr + v_y * v_irb;
      zn = fmin(fmax(zn, v_lb), v_ub);
      const double dy = v_rb * (zr - zn);
      if (keep_steps) {
        dxs[vi] = xn - v_x;
        dyb[vi] = dy;
      }
      v_x = xn;
      v_z = zn;
      v_y += dy;
    }
    __syncthreads();
    PROF_ADD(3);
  }
  if (has_var) {
    q.x[vi] = v_x;
    q.zb[vi] = v_z;
    q.yb[vi] = v_y;
  }
  __syncthreads();
}

// The block of iterations for systems factored in their partition-inverse form (PinvPlan: short trajectories, QP rows in
// shared memory).  As admm_block_fast — shared-memory offsets, scalars in locals, the thread's variable in registers for
// the whole block, preloaded contribution addresses — with the two-step solve, and WARP SPECIALISED: warps 0-5 own the
// partition rows (each thread its row of PI, 3 NB doubles, in registers), warps 6-7 own the QP rows; both take part in the
// separator rows of step A and own their variables.  The two paths never hold each other's state, so neither spills:
// with the 227 KB shared-memory carve-out L1 is a few KB and every spilled register costs an L2 round trip per
// iteration (measured: the single-path version of this block ran slower than the cyclic reduction).  The paths meet at
// `bar.sync 0` (four per iteration), which counts arrivals and does not care where they come from.
template <int NB, int PAIR>
__device__ __noinline__ void admm_block_pinv(const QpCtx& q, const double rho_aux_in, const int n_iter, const int keep_last) {
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  constexpr int kPre = 8;  // column entries whose addresses are kept in registers
  constexpr int QN = 3 * NB;
  constexpr int kRowThreads = 64;  // warps 6-7
  extern __shared__ double sm[];
#ifdef TB200_PROFILE
  const long long prof_entry_ = clock64();
#endif
  const int tid = q.tid, N = q.N, Np = q.Np, nrows = q.nrows, RS = q.RS;
  const double sigma = q.sigma, alpha = q.alpha, oma = 1.0 - q.alpha, rho = q.rho, rho_eq = q.rho_eq, rho_aux = rho_aux_in;
  const double inv_rho_aux = 1.0 / rho_aux, inv_rho = 1.0 / rho, inv_rho_eq = 1.0 / rho_eq;
  double* const v1 = sm + (q.v1 - q.smbase);
  double* const w = sm + (q.w - q.smbase);
  double* const rows = sm + (q.rows - q.smbase);
  const int* const rints = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.rints) - q.smbase));
  const int* const colent = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.colent) - q.smbase));
  double* const dxs = q.scratch;
  double* const dyb = q.scratch + Np;
  // ---- roles in the solve
  const int M = q.M, PR = q.pl.PR, nS = q.pl.nS, ZS = q.pl.ZS, HO = q.pl.HO, WS = q.pl.WS;
  const double* const fbase = sm + (q.SA - q.smbase);
  const bool upper = tid >= kQpThreads - kRowThreads;      // warps 6-7: the QP rows
  const bool prow = tid < PR;                              // a partition row (PR <= 192: always in warps 0-5)
  const int pp = prow ? tid / QN : 0, plr = prow ? tid % QN : 0;
  const int pb0 = pp * 4 * NB, pvar = pb0 + plr;           // first variable of the partition, the variable of this row
  const int pn = ((M - 4 * pp) < 3 ? (M - 4 * pp) : 3) * NB;
  const int xl_off = (pp > 0) ? (4 * pp - 1) * NB : 0;     // solutions of the left / right separator in w (absent: W is 0)
  const int xr_off = (4 * pp + 3 < M) ? (4 * pp + 3) * NB : 0;
  const unsigned a_wrow = smem_u32(fbase + q.pl.wo + (prow ? tid : 0) * WS);
  const unsigned a_b = smem_u32(v1 + pb0), a_xl = smem_u32(w + xl_off), a_xr = smem_u32(w + xr_off);
  const bool swork = tid >= PR && tid < PR + 2 * nS;       // half of a separator row of Z
  const int sw = swork ? tid - PR : 0, srow = sw >> 1, half = sw & 1;
  const int svar = (4 * (srow / NB) + 3) * NB + srow % NB;
  const int c0 = half ? HO : 0, c1 = half ? Np : HO;
  const unsigned a_z = smem_u32(fbase + q.pl.zo + srow * ZS), a_v1 = smem_u32(v1);
  // ---- this thread's variable
  const bool has_var = tid < N;
  const int vi = has_var ? tid : 0;
  const double v_beta = q.beta[vi], v_lb = q.lbs[vi], v_ub = q.ubs[vi], v_qs = q.qs[vi];
  const bool v_eq = v_ub - v_lb < kRhoTol;
  const double v_rb = v_eq ? rho_eq : rho, v_irb = v_eq ? inv_rho_eq : inv_rho;
  double v_x = q.x[vi], v_z = q.zb[vi], v_y = q.yb[vi];
  double v_dx = 0.0, v_dy = 0.0;  // the last iteration's steps (keep_last)
  const int e0 = has_var ? q.colptr[vi] : 0, e1 = has_var ? q.colptr[vi + 1] : 0;
  // a word that always reads 0.0 (the unused last scalar slot of the factorisation scratch)
  double* const zero_slot = sm + (q.flag - q.smbase) + 7;
  if (tid == 0) *zero_slot = 0.0;
  int ea[kPre];
#pragma unroll
  for (int k = 0; k < kPre; ++k) {
    const int e = e0 + k;
    const int ent = (e < e1) ? colent[e] : -1;
    ea[k] = (ent >= 0) ? static_cast<int>(rows - sm) + (ent >> 5) * RS + (2 * CNc + R_NF) + (ent & 31)
                       : static_cast<int>(zero_slot - sm);
  }
  auto bar = []() { asm volatile("bar.sync 0;" ::: "memory"); };
  // right-hand side  sigma x - q + A'(rho z - y): the variable's own part from registers, the rows left their terms behind
  auto build_rhs = [&]() {
    double s = 0.0;
    if (has_var) {
      s = sigma * v_x - v_qs + v_beta * (v_rb * v_z - v_y);
      double c[kPre];
#pragma unroll
      for (int k = 0; k < kPre; ++k) c[k] = sm[ea[k]];
      // (a fixed pairwise order: the eight loads are in flight together instead of one load per dependent add)
      s += ((c[0] + c[1]) + (c[2] + c[3])) + ((c[4] + c[5]) + (c[6] + c[7]));
      for (int e = e0 + kPre; e < e1; ++e) {
        const int ent = colent[e];
        s += rows[(ent >> 5) * RS + (2 * CNc + R_NF) + (ent & 31)];
      }
    }
    if (tid < Np) v1[tid] = s;
  };
  // step A for a separator worker: its half of x_s = Z b; the two halves of a row sit in neighbouring lanes
  auto sep_half = [&]() {
    double zs = 0.0;
    if (swork) {
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int c = c0;
      unsigned az = a_z + c0 * 8, ab = a_v1 + c0 * 8;
#pragma unroll 2
      for (; c + 8 <= c1; c += 8, az += 64, ab += 64) {
        const double2 z0 = lds_v2_at(az), z1 = lds_v2_at(az + 16), z2 = lds_v2_at(az + 32), z3 = lds_v2_at(az + 48);
        const double2 b0 = lds_v2_at(ab), b1 = lds_v2_at(ab + 16), b2 = lds_v2_at(ab + 32), b3 = lds_v2_at(ab + 48);
        s0 += z0.x * b0.x; s1 += z0.y * b0.y; s2 += z1.x * b1.x; s3 += z1.y * b1.y;
        s0 += z2.x * b2.x; s1 += z2.y * b2.y; s2 += z3.x * b3.x; s3 += z3.y * b3.y;
      }
      for (; c < c1; c += 2, az += 16, ab += 16) {
        const double2 z0 = lds_v2_at(az), b0 = lds_v2_at(ab);
        s0 += z0.x * b0.x; s1 += z0.y * b0.y;
      }
      zs = (s0 + s1) + (s2 + s3);
    }
    zs += __shfl_xor_sync(0xffffffffu, zs, 1);
    if (swork && half == 0) w[svar] = zs;
  };
  // the thread's variable and its bound row after the solve
  auto var_update = [&](const bool keep_steps) {
    if (has_var) {
      const double xt = w[vi];
      const double xn = alpha * xt + oma * v_x;
      const double zr = alpha * (v_beta * xt) + oma * v_z;
      double zn = zr + v_y * v_irb;
      zn = fmin(fmax(zn, v_lb), v_ub);
      const double dy = v_rb * (zr - zn);
      if (keep_steps) {
        v_dx = xn - v_x;
        v_dy = dy;
        dxs[vi] = v_dx;
        dyb[vi] = v_dy;
      }
      v_x = xn;
      v_z = zn;
      v_y += dy;
    }
  };

  if (!upper) {
    // ================= warps 0-5: partition rows (PI row in registers), separator halves, variables
    double pi[QN];
#pragma unroll
    for (int j = 0; j < QN; ++j) pi[j] = prow ? q.pi_g[j * PR + tid] : 0.0;
    bar();  // (the entry pass of the row warps)
#ifdef TB200_PROFILE
    if (tid == 0) atomicAdd(&g_prof[21], (unsigned long long)(clock64() - prof_entry_));
#endif
    for (int it = 0; it < n_iter; ++it) {
      const bool keep_steps = keep_last && it == n_iter - 1;
      { PROF_T0(); build_rhs(); PROF_ADD(1); }
      {
        PROF_T0();
        PROF_CHK_T0();
        bar();  // the right-hand side is complete
        PROF_CHK(4);
        double y = 0.0;
        if (prow) {  // step A: y = PI b_p
          double y0 = 0.0, y1 = 0.0;
#pragma unroll
          for (int j = 0; j < QN; j += 2) {
            double2 bb = make_double2(0.0, 0.0);
            if (j < pn) bb = lds_v2_at(a_b + j * 8);
            y0 += pi[j] * bb.x;
            y1 += pi[j + 1] * bb.y;
          }
          y = y0 + y1;
        }
        sep_half();
        PROF_CHK(14);
        bar();
        PROF_CHK(15);
        if (prow) {  // step B: x_p = y - W [x_left; x_right]
          double t0 = 0.0, t1 = 0.0;
#pragma unroll
          for (int t = 0; t < NB; t += 2) {
            const double2 wl = lds_v2_at(a_wrow + t * 8), wr = lds_v2_at(a_wrow + (NB + t) * 8);
            const double2 xl = lds_v2_at(a_xl + t * 8), xr = lds_v2_at(a_xr + t * 8);
            t0 += wl.x * xl.x + wr.x * xr.x;
            t1 += wl.y * xl.y + wr.y * xr.y;
          }
          w[pvar] = y - (t0 + t1);
        }
        bar();
        PROF_CHK(9);
        PROF_ADD(2);
      }
      {
        PROF_T0();
        var_update(keep_steps);
        bar();
        PROF_ADD(3);
      }
    }
  } else {
    // ================= warps 6-7: the QP rows, separator halves, variables
    // entry pass: aux right-hand sides, row multipliers and contributions from the current row state
    for (int r = kQpThreads - 1 - tid; r < nrows; r += kRowThreads)
      admm_row_entry<CNc>(rows + r * RS, rows + r * RS + 2 * CNc, sigma, rho_aux);
    bar();
    for (int it = 0; it < n_iter; ++it) {
      const bool keep_steps = keep_last && it == n_iter - 1;
      build_rhs();
      bar();
      sep_half();
      bar();
      bar();  // (step B of the partition warps)
      // rows: back-substitute aux, relax, project, dual update, and the multipliers for the next solve
      for (int r = kQpThreads - 1 - tid; r < nrows; r += kRowThreads)
        admm_row_update<CNc>(rows + r * RS, rows + r * RS + 2 * CNc, rints + r * RI_NINTS, w, sigma, alpha, oma, rho_aux,
                             inv_rho_aux);
      var_update(keep_steps);
      bar();
    }
  }
  if (has_var) {
    q.x[vi] = v_x;
    q.zb[vi] = v_z;
    q.yb[vi] = v_y;
  }
  __syncthreads();
  if (keep_last == 2) {
    // ---- the terms of the termination check at the end of the block, in one pass (qp_solve_block reduces them where
    // it needs them, fused_q) instead of the generic passes of info_pass, the certificates and the guess hash, with their ten-odd
    // barriers.  Variables: their row of P x (p_matvec's order), A'y (scatter_columns' order), their norm terms, the
    // certificates' first stages and the guess hash, from the state in registers; rows on warps 6-7.  The norms are
    // maxima and the hash a wrapping sum, so they come out exactly as from the generic passes; the two floating-point
    // sums of the certificates (u'dy+ + l'dy- and q'dx) are added in another order than there.
    double m[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double pa[3] = {0.0, 0.0, 0.0}, da[2] = {0.0, 0.0};
    unsigned long long h = 0ull;
    const double* const xs = sm + (q.x - q.smbase);
    const double* const Dz = sm + (q.Dz - q.smbase);
    if (has_var) {
      const double px = p_row<NB>(q, vi, Dz, xs);
      double aty = v_beta * v_y;
      for (int e = e0; e < e1; ++e) {
        const int ent = colent[e];
        const double* R = rows + (ent >> 5) * RS;
        aty += R[CNc + (ent & 31)] * R[2 * CNc + R_Y];
      }
      const double dz = Dz[vi];
      info_var_terms(dz, v_beta, v_x, v_z, aty, px, v_qs, m);
      pinf_var_terms(v_beta / dz, v_ub, v_lb, v_dy, pa);
      da[0] = fmax(da[0], fabs(dz * v_dx));
      da[1] += v_qs * v_dx;
      h += guess_var_hash(v_z, v_y, v_lb, v_ub, vi, nrows);
    }
    if (upper) {
      for (int r = kQpThreads - 1 - tid; r < nrows; r += kRowThreads) {
        const double* R = rows + r * RS;
        double* F = rows + r * RS + 2 * CNc;
        const int* I = rints + r * RI_NINTS;
        const double ax = row_dot<CNc>(q, R, I, xs) + F[R_U0] * F[R_XA0] + F[R_U1] * F[R_XA1];
        info_row_terms(F, ax, m);
        pinf_row_terms(F, I[RI_AUX], pa);
        dinf_row_terms(F, da);
        h += guess_row_hash(F, I, r, nrows, N);
      }
    }
    // warp partials, reduced like block_reduce
    double vals[kChkHash] = {m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8], m[9], m[10], m[11], m[12], m[13],
                             pa[0], pa[1], pa[2], da[0], da[1]};
    static_assert(CHK_PA0 == 14 && CHK_DA1 == 18, "vals[] follows ChkQ");
    __syncwarp();
#pragma unroll
    for (int k = 0; k < kChkHash; ++k) {
      double v = vals[k];
      if ((kChkSumMask >> k) & 1u) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      } else {
        v = warp_max_norm(v);
      }
      vals[k] = v;
    }
    for (int off = 16; off > 0; off >>= 1) h += __shfl_xor_sync(0xffffffffu, h, off);
    if ((tid & 31) == 0) {
      double* const chk = sm + (q.tmp - q.smbase);
      const int wid = tid >> 5;
#pragma unroll
      for (int k = 0; k < kChkHash; ++k) chk[k * 8 + wid] = vals[k];
      reinterpret_cast<unsigned long long*>(chk + kChkHash * 8)[wid] = h;
    }
    __syncthreads();
  }
}

// The block of iterations for QPs whose rows do not fit shared memory (configs[3] at 50 waypoints: ~370 rows of 14
// coefficients; configs[4]).  Their row records live in global memory, 98 doubles apart: a warp that works on 32 rows
// touches 32 different sectors with every field it loads (4x the bytes it uses), and the right-hand side gathers the rows'
// contributions through two dependent loads per entry.  So for the duration of a block the fields the loop needs are
// copied into a COLUMN-MAJOR block of this CTA (field f of row r at soa[f * RSd + r]: a warp's load of a field is one
// contiguous 256 bytes, all loads of a row independent), the contributions go to ct[e] in column-entry order (the
// right-hand side of variable i adds ct[colptr[i] .. colptr[i+1]) - contiguous, addresses known up front), and the row
// state goes back to the records at the end.  Same arithmetic, operation for operation, as admm_block.
enum SoaF { S_U0 = 0, S_U1, S_B0, S_B1, S_LO, S_UP, S_QA0, S_QA1, S_WRR, S_IWRR, S_G0, S_G1, S_IDEN, S_UPA0, S_UPA1,
            S_Z, S_Y, S_XA0, S_XA1, S_ZA0, S_ZA1, S_YA0, S_YA1, S_RA0, S_RA1, S_AS };  // S_AS: CN scaled coefficients follow
__host__ __device__ inline size_t qp_soa_doubles(int max_rows, int CN) {
  const size_t rsd = (static_cast<size_t>(max_rows) + 31) & ~static_cast<size_t>(31);
  return rsd * (S_AS + CN) + (rsd * (3 + CN) + 1) / 2 + static_cast<size_t>(max_rows) * CN + 8;
}
template <int NB, int PAIR>
__device__ __noinline__ void admm_block_soa(const QpCtx& q, const double rho_aux_in, const int n_iter, const int keep_last) {
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  const int N = q.N, Np = q.Np, tid = q.tid, nrows = q.nrows;
  const double sigma = q.sigma, alpha = q.alpha, oma = 1.0 - q.alpha, rho = q.rho, rho_eq = q.rho_eq, rho_aux = rho_aux_in;
  const double inv_rho_aux = 1.0 / rho_aux, inv_rho = 1.0 / rho, inv_rho_eq = 1.0 / rho_eq;
  double* const dxs = q.scratch;
  double* const dyb = q.scratch + Np;
  const int RSd = (nrows + 31) & ~31;
  double* const sd = q.soa;                                                      // [S_AS + CNc][RSd]
  int* const si = reinterpret_cast<int*>(sd + static_cast<size_t>(RSd) * (S_AS + CNc));  // [3 + CNc][RSd]: base, stride, last, entry of k
  double* const ct = sd + static_cast<size_t>(RSd) * (S_AS + CNc) + (static_cast<size_t>(RSd) * (3 + CNc) + 1) / 2 + 1;
  const int nnz = q.colptr[Np];
  PROF_T0();
  // ---- entry: entry index of every (row, coefficient); fields of every row; contributions of the current state
  for (int i = tid; i < N; i += kQpThreads)
    for (int e = q.colptr[i]; e < q.colptr[i + 1]; ++e) {
      const int ent = q.colent[e];
      si[(3 + (ent & 31)) * RSd + (ent >> 5)] = e;
    }
  for (int e = tid; e < nnz; e += kQpThreads) ct[e] = 0.0;
  __syncthreads();
  for (int r = tid; r < nrows; r += kQpThreads) {
    const double* R = q.R(r);
    const double* F = q.F(r);
    const int* I = q.I(r);
    const int cnt = I[RI_CNT];
    si[r] = I[RI_BASE];
    si[RSd + r] = I[RI_STRIDE];
    si[2 * RSd + r] = cnt - 1;
    sd[S_U0 * RSd + r] = F[R_U0]; sd[S_U1 * RSd + r] = F[R_U1]; sd[S_B0 * RSd + r] = F[R_B0]; sd[S_B1 * RSd + r] = F[R_B1];
    sd[S_LO * RSd + r] = F[R_LO]; sd[S_UP * RSd + r] = F[R_UP]; sd[S_QA0 * RSd + r] = F[R_QA0]; sd[S_QA1 * RSd + r] = F[R_QA1];
    sd[S_WRR * RSd + r] = F[R_WRR]; sd[S_IWRR * RSd + r] = F[R_IWRR]; sd[S_G0 * RSd + r] = F[R_G0]; sd[S_G1 * RSd + r] = F[R_G1];
    sd[S_IDEN * RSd + r] = F[R_IDEN];
    sd[S_UPA0 * RSd + r] = kOsqpInf * F[R_EA0]; sd[S_UPA1 * RSd + r] = kOsqpInf * F[R_EA1];
    sd[S_Z * RSd + r] = F[R_Z]; sd[S_Y * RSd + r] = F[R_Y]; sd[S_XA0 * RSd + r] = F[R_XA0]; sd[S_XA1 * RSd + r] = F[R_XA1];
    sd[S_ZA0 * RSd + r] = F[R_ZA0]; sd[S_ZA1 * RSd + r] = F[R_ZA1]; sd[S_YA0 * RSd + r] = F[R_YA0]; sd[S_YA1 * RSd + r] = F[R_YA1];
    const double s0 = F[R_WRR] * F[R_Z] - F[R_Y];
    const double ra0 = sigma * F[R_XA0] - F[R_QA0] + F[R_U0] * s0 + F[R_B0] * (rho_aux * F[R_ZA0] - F[R_YA0]);
    const double ra1 = sigma * F[R_XA1] - F[R_QA1] + F[R_U1] * s0 + F[R_B1] * (rho_aux * F[R_ZA1] - F[R_YA1]);
    sd[S_RA0 * RSd + r] = ra0;
    sd[S_RA1 * RSd + r] = ra1;
    const double cf = row_reduce_coef(F, ra0, ra1, s0);
#pragma unroll
    for (int k = 0; k < CNc; ++k) {
      const double a = R[CNc + k];
      sd[(S_AS + k) * RSd + r] = a;
      if (k < cnt) ct[si[(3 + k) * RSd + r]] = a * cf;
    }
  }
  __syncthreads();
  PROF_ADD(0);
  for (int it = 0; it < n_iter; ++it) {
    const bool keep_steps = keep_last && it == n_iter - 1;
    // right-hand side  sigma x - q + A'(rho z - y)
    long long pt_ = 0;
#ifdef TB200_PROFILE
    pt_ = clock64();
#define PROF_SOA(slot) do { const long long n_ = clock64(); if (tid == 0) atomicAdd(&g_prof[slot], (unsigned long long)(n_ - pt_)); pt_ = n_; } while (0)
#else
#define PROF_SOA(slot) (void)pt_
#endif
    for (int i = tid; i < Np; i += kQpThreads) {
      double s = 0.0;
      if (i < N) {
        const double rb = (q.ubs[i] - q.lbs[i] < kRhoTol) ? rho_eq : rho;
        s = sigma * q.x[i] - q.qs[i] + q.beta[i] * (rb * q.zb[i] - q.yb[i]);
        const int e1 = q.colptr[i + 1];
        for (int e = q.colptr[i]; e < e1; ++e) s += ct[e];
      }
      q.v1[i] = s;
    }
    PROF_SOA(1);
    bcr_solve<NB>(q, q.v1, q.w);
    PROF_SOA(2);
    // rows
    for (int r = tid; r < nrows; r += kQpThreads) {
      const int base = si[r], stride = si[RSd + r], last = si[2 * RSd + r];
      double as[CNc];
#pragma unroll
      for (int k = 0; k < CNc; ++k) as[k] = sd[(S_AS + k) * RSd + r];
      const double U0 = sd[S_U0 * RSd + r], U1 = sd[S_U1 * RSd + r], B0 = sd[S_B0 * RSd + r], B1 = sd[S_B1 * RSd + r];
      const double LO = sd[S_LO * RSd + r], UP = sd[S_UP * RSd + r], QA0 = sd[S_QA0 * RSd + r], QA1 = sd[S_QA1 * RSd + r];
      const double Wr = sd[S_WRR * RSd + r], IWRR = sd[S_IWRR * RSd + r], G0 = sd[S_G0 * RSd + r], G1 = sd[S_G1 * RSd + r];
      const double iden = sd[S_IDEN * RSd + r], UPA0 = sd[S_UPA0 * RSd + r], UPA1 = sd[S_UPA1 * RSd + r];
      const double Z = sd[S_Z * RSd + r], Y = sd[S_Y * RSd + r], XA0 = sd[S_XA0 * RSd + r], XA1 = sd[S_XA1 * RSd + r];
      const double ZA0 = sd[S_ZA0 * RSd + r], ZA1 = sd[S_ZA1 * RSd + r], YA0 = sd[S_YA0 * RSd + r], YA1 = sd[S_YA1 * RSd + r];
      const double ra0o = sd[S_RA0 * RSd + r], ra1o = sd[S_RA1 * RSd + r];
      double zeta = 0.0;
#pragma unroll
      for (int k = 0; k < CNc; ++k) zeta += as[k] * q.w[base + min(k, last) * stride];
      // row_backsub
      const double a0 = (G1 * (ra0o - Wr * U0 * zeta) + Wr * U1 * (U1 * ra0o - U0 * ra1o)) * iden;
      const double a1 = (G0 * (ra1o - Wr * U1 * zeta) + Wr * U0 * (U0 * ra1o - U1 * ra0o)) * iden;
      const double zt = zeta + U0 * a0 + U1 * a1;
      const double zr = alpha * zt + oma * Z;
      double zn = zr + Y * IWRR;
      zn = fmin(fmax(zn, LO), UP);
      const double dy = Wr * (zr - zn);
      const double yn = Y + dy;
      const double s = Wr * zn - yn;
      // aux 0
      const double xn0 = alpha * a0 + oma * XA0;
      const double zra0 = alpha * (B0 * a0) + oma * ZA0;
      double z20 = zra0 + YA0 * inv_rho_aux;
      z20 = fmin(fmax(z20, 0.0), UPA0);
      const double dya0 = rho_aux * (zra0 - z20);
      const double yan0 = YA0 + dya0;
      const double ra0 = sigma * xn0 - QA0 + U0 * s + B0 * (rho_aux * z20 - yan0);
      // aux 1
      const double xn1 = alpha * a1 + oma * XA1;
      const double zra1 = alpha * (B1 * a1) + oma * ZA1;
      double z21 = zra1 + YA1 * inv_rho_aux;
      z21 = fmin(fmax(z21, 0.0), UPA1);
      const double dya1 = rho_aux * (zra1 - z21);
      const double yan1 = YA1 + dya1;
      const double ra1 = sigma * xn1 - QA1 + U1 * s + B1 * (rho_aux * z21 - yan1);
      // row_reduce_coef
      const double cf = s - Wr * (U0 * ra0 * G1 + U1 * ra1 * G0) * iden;
      sd[S_Z * RSd + r] = zn; sd[S_Y * RSd + r] = yn; sd[S_XA0 * RSd + r] = xn0; sd[S_XA1 * RSd + r] = xn1;
      sd[S_ZA0 * RSd + r] = z20; sd[S_ZA1 * RSd + r] = z21; sd[S_YA0 * RSd + r] = yan0; sd[S_YA1 * RSd + r] = yan1;
      sd[S_RA0 * RSd + r] = ra0; sd[S_RA1 * RSd + r] = ra1;
#pragma unroll
      for (int k = 0; k < CNc; ++k)
        if (k <= last) ct[si[(3 + k) * RSd + r]] = as[k] * cf;
      if (it == n_iter - 1) {  // the state (and, for the certificates, the last steps) go back to the row record
        double* F = q.F(r);
        F[R_Z] = zn; F[R_Y] = yn; F[R_DY] = dy;
        F[R_XA0] = xn0; F[R_XA1] = xn1; F[R_DXA0] = xn0 - XA0; F[R_DXA1] = xn1 - XA1;
        F[R_ZA0] = z20; F[R_ZA1] = z21; F[R_YA0] = yan0; F[R_YA1] = yan1; F[R_DYA0] = dya0; F[R_DYA1] = dya1;
        F[R_RA0] = ra0; F[R_RA1] = ra1; F[R_COEF] = cf;
      }
    }
    // trajectory variables and their bound rows
    for (int i = tid; i < N; i += kQpThreads) {
      const double beta = q.beta[i];
      const double lb = q.lbs[i], ub = q.ubs[i];
      const bool beq = ub - lb < kRhoTol;
      const double rb = beq ? rho_eq : rho, irb = beq ? inv_rho_eq : inv_rho;
      const double xt = q.w[i];
      const double xn = alpha * xt + oma * q.x[i];
      const double zr = alpha * (beta * xt) + oma * q.zb[i];
      double zn = zr + q.yb[i] * irb;
      zn = fmin(fmax(zn, lb), ub);
      const double dy = rb * (zr - zn);
      if (keep_steps) {
        dxs[i] = xn - q.x[i];
        dyb[i] = dy;
      }
      q.x[i] = xn;
      q.zb[i] = zn;
      q.yb[i] += dy;
    }
    __syncthreads();
    PROF_SOA(3);
  }
}

// Ruiz equilibration (scale_data of OSQP [EXT]); leaves the scaled view of every row in its record and the
// scaled trajectory cost / bounds in q.qs / q.lbs / q.ubs, Dz (global) / beta (shared).
__device__ inline void qp_scale(QpCtx& q, const QpSettings& st, int n_aux_total) {
  double *qs = q.qs, *lbs = q.lbs, *ubs = q.ubs;
  const int N = q.N, tid = q.tid, HB = 2 * q.D, W = HB + 1;
  double* Eb = q.zb;  // bound-row scalings live in zb during scaling
  q.c = 1.0;
  for (int i = tid; i < q.Np; i += kQpThreads) {
    q.Dz[i] = 1.0;
    Eb[i] = 1.0;
  }
  for (int r = tid; r < q.nrows; r += kQpThreads) {
    double* F = q.F(r);
    F[R_E] = F[R_DA0] = F[R_DA1] = F[R_EA0] = F[R_EA1] = 1.0;
  }
  __syncthreads();
  for (int pass = 0; pass < st.scaling; ++pass) {
    // row norms (one thread per row) -> E_temp in R_RA0; aux column / bound-row scalings updated in place
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      double* R = q.R(r);
      double* F = q.F(r);
      const int* I = q.I(r);
      const int base = I[RI_BASE], cnt = I[RI_CNT], stride = I[RI_STRIDE], aux = I[RI_AUX];
      const double E = F[R_E];
      double rn = 0.0;
      for (int k = 0; k < cnt; ++k) rn = fmax(rn, fabs(E * R[k] * q.Dz[base + k * stride]));
      double dt0 = 1.0, dt1 = 1.0, et0 = 1.0, et1 = 1.0;
      if (aux >= 1) {
        const double ua = fabs(E * F[R_DA0]), ba = fabs(F[R_EA0] * F[R_DA0]);
        rn = fmax(rn, ua);
        dt0 = 1.0 / sqrt(limit_scaling(fmax(ua, ba)));
        et0 = 1.0 / sqrt(limit_scaling(ba));
      }
      if (aux == 2) {
        const double ua = fabs(E * F[R_DA1]), ba = fabs(F[R_EA1] * F[R_DA1]);
        rn = fmax(rn, ua);
        dt1 = 1.0 / sqrt(limit_scaling(fmax(ua, ba)));
        et1 = 1.0 / sqrt(limit_scaling(ba));
      }
      F[R_RA0] = 1.0 / sqrt(limit_scaling(rn));
      F[R_RA1] = E;  // E before this pass (the column pass below must still see the old value)
      F[R_DA0] *= dt0;
      F[R_DA1] *= dt1;
      F[R_EA0] *= et0;
      F[R_EA1] *= et1;
    }
    __syncthreads();
    // column norms of [P A'; A 0] restricted to the trajectory variables (one thread per variable)
    for (int i = tid; i < N; i += kQpThreads) {
      double m = 0.0;
      for (int t = 0; t < q.n_band; ++t) {  // (structurally zero band entries cannot raise a norm)
        const int k = q.band_offs[t];
        if (k <= i) m = fmax(m, fabs(q.c * q.Dz[i] * q.Pband[i * W + k] * q.Dz[i - k]));
        if (k >= 1 && i + k < N) m = fmax(m, fabs(q.c * q.Dz[i] * q.Pband[(i + k) * W + k] * q.Dz[i + k]));
      }
      const double bn = fabs(Eb[i] * q.Dz[i]);
      m = fmax(m, bn);
      for (int e = q.colptr[i]; e < q.colptr[i + 1]; ++e) {
        const int ent = q.colent[e], r = ent >> 5, k = ent & 31;
        const double* R = q.R(r);
        m = fmax(m, fabs(R[2 * q.CN + R_RA1] * R[k] * q.Dz[i]));
      }
      q.v1[i] = 1.0 / sqrt(limit_scaling(m));
      Eb[i] *= 1.0 / sqrt(limit_scaling(bn));
    }
    __syncthreads();
    for (int i = tid; i < N; i += kQpThreads) q.Dz[i] *= q.v1[i];
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      double* F = q.F(r);
      F[R_E] = F[R_RA1] * F[R_RA0];
    }
    __syncthreads();
    // cost normalisation: mean column inf-norm of the scaled P over ALL n variables (aux columns are 0)
    double csum = 0.0, qn = 0.0;
    for (int i = tid; i < N; i += kQpThreads) {
      double m = 0.0;
      for (int t = 0; t < q.n_band; ++t) {  // (structurally zero band entries cannot raise a norm)
        const int k = q.band_offs[t];
        if (k <= i) m = fmax(m, fabs(q.c * q.Dz[i] * q.Pband[i * W + k] * q.Dz[i - k]));
        if (k >= 1 && i + k < N) m = fmax(m, fabs(q.c * q.Dz[i] * q.Pband[(i + k) * W + k] * q.Dz[i + k]));
      }
      csum += m;
      qn = fmax(qn, fabs(q.c * q.Dz[i] * qs[i]));
    }
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      const double* F = q.F(r);
      const int aux = q.I(r)[RI_AUX];
      if (aux >= 1) qn = fmax(qn, fabs(q.c * F[R_DA0] * F[R_W]));
      if (aux == 2) qn = fmax(qn, fabs(q.c * F[R_DA1] * F[R_W]));
    }
    double red2[2] = {csum, qn};
    block_reduce<2, 0x1u>(q, red2);
    const double mean = limit_scaling(red2[0] / static_cast<double>(N + n_aux_total));
    q.c *= 1.0 / fmax(mean, limit_scaling(red2[1]));
  }
  q.cinv = 1.0 / q.c;
  for (int i = tid; i < q.Np; i += kQpThreads) {
    if (i < N) {
      qs[i] = q.c * q.Dz[i] * qs[i];
      lbs[i] *= Eb[i];
      ubs[i] *= Eb[i];
      q.beta[i] = Eb[i] * q.Dz[i];
    } else {
      qs[i] = 0.0; lbs[i] = -1.0; ubs[i] = 1.0; q.beta[i] = 1.0; q.Dz[i] = 1.0;
    }
  }
  // scaled view of every row (padding coefficients stay exactly 0)
  for (int r = tid; r < q.nrows; r += kQpThreads) {
    double* R = q.R(r);
    double* F = q.F(r);
    const int* I = q.I(r);
    const int aux = I[RI_AUX];
    const double E = F[R_E];
    for (int k = 0; k < q.CN; ++k) R[q.CN + k] = E * R[k] * q.Dz[row_var(I, k)];
    F[R_U0] = F[R_U1] = F[R_B0] = F[R_B1] = F[R_QA0] = F[R_QA1] = 0.0;
    F[R_UP] = -F[R_C] * E;
    if (aux == AUX_HINGE) {
      F[R_U0] = -E * F[R_DA0];
      F[R_B0] = F[R_EA0] * F[R_DA0];
      F[R_QA0] = q.c * F[R_DA0] * F[R_W];
      F[R_LO] = -kOsqpInf * E;
      F[R_RHO] = 0.0;
    } else {
      if (aux == AUX_ABS) {
        F[R_U0] = E * F[R_DA0];
        F[R_U1] = -E * F[R_DA1];
        F[R_B0] = F[R_EA0] * F[R_DA0];
        F[R_B1] = F[R_EA1] * F[R_DA1];
        F[R_QA0] = q.c * F[R_DA0] * F[R_W];
        F[R_QA1] = q.c * F[R_DA1] * F[R_W];
      }
      F[R_LO] = F[R_UP];
      F[R_RHO] = 1.0;
    }
  }
  __syncthreads();
}

// The refinement passes of the polish (qp_solve_block: polish_refine) for the partition-inverse layout: rows, row
// index table, column entries, vectors and the cyclic-reduction factor of the polish system all in shared memory and
// addressed as offsets, each variable's state in the registers of thread `i`, the rows on warps 6-7, and the solve
// through fixed per-thread roles (bcr_solve_sm: the same products and sums as bcr_solve).  Its own function, called
// through a pointer, for the reason of admm_block (§4.3 of DESIGN.md): inlined into qp_step, these passes ran on the
// registers the solver's state leaves free and spilled.  Every value is the expression of polish_refine in its order,
// so the polished point is bit for bit the same.  Needs Np <= kQpThreads and solve roles that fit the CTA.
struct PolishRes {
  double p_pri, p_dua, bad;  // max primal residual, max dual residual (scaled by c), wrongly signed multipliers
};
template <int NB, int PAIR>
__device__ __noinline__ PolishRes polish_passes(const QpCtx& q, const int refine_iter) {
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  constexpr int kRowThreads = 64;  // warps 6-7
  extern __shared__ double sm[];
  const int tid = q.tid, N = q.N, Np = q.Np, nrows = q.nrows, RS = q.RS;
  double* const rows = sm + (q.rows - q.smbase);
  const int* const rints = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.rints) - q.smbase));
  const int* const colent = reinterpret_cast<const int*>(sm + (reinterpret_cast<const double*>(q.colent) - q.smbase));
  double* const xs = sm + (q.x - q.smbase);
  double* const v1 = sm + (q.v1 - q.smbase);
  double* const w = sm + (q.w - q.smbase);
  const double* const Dz = sm + (q.Dz - q.smbase);
  const SolveRoles roles = solve_roles<NB>(q);
  const bool upper = tid >= kQpThreads - kRowThreads;
  // ---- this thread's variable (the polish weight's sign in zb: + upper bound active, - lower, 0 free)
  const bool has_var = tid < N;
  const int vi = has_var ? tid : 0;
  const double v_beta = q.beta[vi], v_lb = q.lbs[vi], v_ub = q.ubs[vi], v_qs = q.qs[vi], v_dz = Dz[vi], v_zb = q.zb[vi];
  const double v_w = fabs(v_zb), v_bnd = v_zb > 0 ? v_ub : v_lb;
  const int e0 = has_var ? q.colptr[vi] : 0, e1 = has_var ? q.colptr[vi + 1] : 0;
  double v_x = q.x[vi], v_y = q.yb[vi];
  const double cinv = q.cinv;
  __syncthreads();
  for (int it = 0; it <= refine_iter + 1; ++it) {
    const bool last = (it == refine_iter + 1);  // final pass: pending dual update + residuals only
    double mm[3] = {0.0, 0.0, 0.0};             // m_pri (max), m_dua (max), bad signs (sum)
    double px = 0.0;
    if (has_var) px = p_row<NB>(q, vi, Dz, xs);  // (P xq)_i
    if (upper) {
      for (int r = kQpThreads - 1 - tid; r < nrows; r += kRowThreads) {
        const double* R = rows + r * RS;
        double* F = rows + r * RS + 2 * CNc;
        const int* I = rints + r * RI_NINTS;
        const int naux = I[RI_AUX];
        const double Wr = F[R_WRR];
        const double ax = row_dot<CNc>(q, R, I, xs) + F[R_U0] * F[R_PX0] + F[R_U1] * F[R_PX1];
        const double py = F[R_PY] + ((it > 0) ? Wr * (ax - F[R_PB]) : 0.0);
        const double e = py + (last ? 0.0 : Wr * (ax - F[R_PB]));
        const double zc = fmin(fmax(ax, F[R_LO]), F[R_UP]);
        mm[0] = fmax(mm[0], fabs((ax - zc) / F[R_E]));
        mm[2] += (last && Wr != 0.0 && naux == AUX_HINGE && py < -kVerifyTol) ? 1.0 : 0.0;  // upper active needs y >= 0
        double pya[2], ra[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const double bb = F[R_B0 + k], u = F[R_U0 + k], qa = F[R_QA0 + k];
          const double wa = fabs(F[R_PWA0 + k]);
          const double axb = bb * F[R_PX0 + k];
          pya[k] = F[R_PYA0 + k] + ((it > 0) ? wa * axb : 0.0);
          const double ea = pya[k] + (last ? 0.0 : wa * axb);
          mm[0] = fmax(mm[0], fabs((axb - fmax(axb, 0.0)) / F[R_EA0 + k]));
          mm[2] += (last && wa != 0.0 && pya[k] > kVerifyTol) ? 1.0 : 0.0;  // aux >= 0 held at 0 needs y <= 0
          mm[1] = fmax(mm[1], fabs((qa + u * py + bb * pya[k]) / F[R_DA0 + k]));
          ra[k] = -qa - u * e - bb * ea;
        }
        F[R_PY] = py;
        F[R_PYA0] = pya[0];
        F[R_PYA1] = pya[1];
        F[R_RA0] = ra[0];
        F[R_RA1] = ra[1];
        F[R_COEF] = last ? py : row_reduce_coef(F, ra[0], ra[1], -e);
      }
    }
    __syncthreads();
    // the variable's column: last pass the dual residual P x + q + A'y, else rd = -(P x + q) - beta (y + W (A x - b))
    // + A' coef (scatter_columns' order)
    if (tid < Np) {
      double s = 0.0;
      if (has_var) {
        s = last ? px + v_qs + v_beta * v_y : -(px + v_qs) - v_beta * (v_y + v_w * (v_beta * v_x - v_bnd));
        for (int e = e0; e < e1; ++e) {
          const int ent = colent[e];
          const double* R = rows + (ent >> 5) * RS;
          s += R[CNc + (ent & 31)] * R[2 * CNc + R_COEF];
        }
        const double ax = v_beta * v_x;
        const double zc = fmin(fmax(ax, v_lb), v_ub);
        mm[0] = fmax(mm[0], fabs((ax - zc) * v_dz / v_beta));
        const bool ineq = last && v_w != 0.0 && (v_ub - v_lb >= kRhoTol);
        mm[2] += (ineq && v_zb > 0 && v_y < -kVerifyTol) ? 1.0 : 0.0;
        mm[2] += (ineq && v_zb < 0 && v_y > kVerifyTol) ? 1.0 : 0.0;
        if (last) mm[1] = fmax(mm[1], fabs(s / v_dz));
      }
      v1[tid] = s;
    }
    if (last) {
      if (has_var) q.yb[vi] = v_y;
      block_reduce<3, 0x4u>(q, mm);
      return PolishRes{mm[0], mm[1] * cinv, mm[2]};
    }
    bcr_solve_sm<NB>(tid, roles, sm, v1, w);  // (begins with a barrier)
    if (upper) {
      for (int r = kQpThreads - 1 - tid; r < nrows; r += kRowThreads) {
        const double* R = rows + r * RS;
        double* F = rows + r * RS + 2 * CNc;
        double a0, a1;
        row_backsub(F, row_dot<CNc>(q, R, rints + r * RI_NINTS, w), a0, a1);
        F[R_PX0] += a0;
        F[R_PX1] += a1;
      }
    }
    if (has_var) {
      const double xn = v_x + w[vi];
      // multiplier update of the variable-bound rows with the new iterate (the rows do theirs at the start of the
      // next pass, where A x is recomputed anyway)
      v_y += v_w * (v_beta * xn - v_bnd);
      v_x = xn;
      xs[vi] = xn;
    }
    __syncthreads();
  }
  return PolishRes{0.0, 0.0, 0.0};  // (not reached)
}

// The QP solve for the calling CTA's trajectory (initial iterate from the warm start or zero).
// Every scalar that steers control flow is derived from block-reduced values, so all threads take the same path.
// REGOK: the register-resident solve may be used (its per-thread factor rows fit the register file: blocks of <= 14).
// fast_passes: the termination checks computed by the partition-inverse block (admm_block_pinv) and the polish
// refinement by polish_passes, where the layout allows.
template <int NB, int PAIR, bool REGOK>
__device__ inline QpOut qp_solve_block(QpCtx& q, const QpSettings& st, bool warm, double warm_rho,
                                       const double* ws_x, const double* ws_yb, const bool fast_passes) {
  // coefficients per (padded) row: D, or 2*D when rows may span two consecutive waypoints (CartVel, cast collision)
  constexpr int CNc = PAIR ? ((NB > 3) ? NB : 3) : ((NB / 2 > 3) ? NB / 2 : 3);
  const int N = q.N, tid = q.tid;
  QpOut out{QPS_UNSOLVED, 0, 0, st.rho, 0, 0, 0, 0, 0, -1, 0, 0};
  double rho;
  double eps_scale;
  int iter, round;
  q.sigma = st.sigma;
  q.alpha = st.alpha;
  {
    rho = warm ? warm_rho : st.rho;
    rho = fmin(fmax(rho, kRhoMin), kRhoMax);
    eps_scale = 1.0;
    iter = 0;
    round = 0;
    q.rho = rho;
    q.rho_eq = kRhoEqOverIneq * rho;
    if (warm) {  // osqp_warm_start: x <- Dinv x, y <- c Einv y, z <- A x
      for (int i = tid; i < q.Np; i += kQpThreads) {
        if (i < N) {
          q.x[i] = ws_x[i] / q.Dz[i];
          q.yb[i] = ws_yb[i] * q.Dz[i] / q.beta[i] * q.c;   // Eb = beta / Dz
          q.zb[i] = q.beta[i] * q.x[i];
        } else {
          q.x[i] = q.yb[i] = q.zb[i] = 0.0;
        }
      }
      __syncthreads();
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        double* R = q.R(r);
        double* F = q.F(r);
        const int naux = q.I(r)[RI_AUX];
        F[R_XA0] = (naux >= 1) ? F[R_XA0] / F[R_DA0] : 0.0;
        F[R_XA1] = (naux == 2) ? F[R_XA1] / F[R_DA1] : 0.0;
        F[R_Y] = F[R_Y] / F[R_E] * q.c;
        F[R_YA0] = (naux >= 1) ? F[R_YA0] / F[R_EA0] * q.c : 0.0;
        F[R_YA1] = (naux == 2) ? F[R_YA1] / F[R_EA1] * q.c : 0.0;
        F[R_Z] = row_dot<CNc>(q, R, q.I(r), q.x) + F[R_U0] * F[R_XA0] + F[R_U1] * F[R_XA1];
        F[R_ZA0] = F[R_B0] * F[R_XA0];
        F[R_ZA1] = F[R_B1] * F[R_XA1];
      }
    } else {
      for (int i = tid; i < q.Np; i += kQpThreads) q.x[i] = q.zb[i] = q.yb[i] = 0.0;
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        double* F = q.F(r);
        F[R_XA0] = F[R_XA1] = F[R_Z] = F[R_Y] = F[R_ZA0] = F[R_ZA1] = F[R_YA0] = F[R_YA1] = 0.0;
      }
    }
    __syncthreads();
  }
  SysW sysw{false, st.sigma, rho};
  bool factor_ok = true;

  // the ADMM block, the fused check and the polish refinement of this QP (QpPlan)
  const QpPlan plan = qp_plan(REGOK, q.pinv, q.rows_smem, q.M, NB, fast_passes);
  const bool use_reg = plan.use_reg;
  const bool use_pinv = plan.use_pinv;
  using BlockFn = void (*)(const QpCtx&, double, int, int);
  const bool fuse = plan.fuse;
  const bool fast_polish = plan.fast_polish;
  // q.tmp holds the fused check's partials of the current iterate: set by a block that computed them, cleared by every
  // factorisation (it reuses q.tmp)
  bool fused_chk = false;
  auto run_block = [&](int n, bool keep_last) {
    fused_chk = fuse && keep_last;
    if constexpr (REGOK) {
      if (use_pinv || use_reg) {
        // (called through pointers: an indirect call follows the standard calling convention, so the block gets the
        // whole register file — saving what it uses of the callee-saved registers at entry — instead of the registers
        // this solver's own state leaves free.  Measured: with a direct call the caller's register allocation squeezes
        // the loop and every level of its solve is scheduled one shared-memory load at a time.)
        BlockFn volatile fn = use_pinv ? &admm_block_pinv<NB, PAIR>
                                       : (q.rows_smem ? &admm_block_fast<NB, PAIR> : &admm_block_soa<NB, PAIR>);
        fn(q, sysw.rho_aux, n, keep_last ? (fuse ? 2 : 1) : 0);
        return;
      }
    }
    // long trajectories / wide blocks: rows in shared memory -> the plain block; rows in global memory -> column-major copy
    BlockFn volatile fn = q.rows_smem ? &admm_block<NB, PAIR> : &admm_block_soa<NB, PAIR>;
    fn(q, sysw.rho_aux, n, keep_last ? 1 : 0);
  };
  // the same for the factorisation (a few calls per QP, tens of thousands of cycles each); the polish system always
  // takes the cyclic reduction (its solves are the generic ones), with warp-local block inversions when the factor is
  // in shared memory (the CTA-wide ones, same values, under TB200_GENERIC_QP_PASSES=1: the reference of the tests)
  using FactorFn = bool (*)(const QpCtx&, const SysW&);
  auto factorize = [&](const SysW& wts) -> bool {
    fused_chk = false;
    FactorFn f = &assemble_factor<NB, false, false>;
    if constexpr (NB <= 16) {
      if (fast_passes && __isShared(q.SA)) f = &assemble_factor<NB, false, true>;
    }
    if constexpr (REGOK) {
      if (use_pinv && !wts.polish) f = &assemble_factor<NB, true, false>;
    }
    FactorFn volatile fn = f;
    return fn(q, wts);
  };
  // A polish factors its own system over Z (the rest of the partition-inverse form lies beyond the cyclic-reduction
  // layout): Z is copied to global memory before and, when the polish fails, copied back — the same bytes a new
  // factorisation of the unchanged ADMM system would produce, at a hundredth of its cost.
  auto stash_z = [&](const bool restore) {
    extern __shared__ double sm[];
    double2* zs = reinterpret_cast<double2*>(sm + (q.SA - q.smbase) + q.pl.zo);
    double2* zg = reinterpret_cast<double2*>(q.z_stash);
    const int n2 = q.pl.nS * q.pl.ZS / 2;
    if (restore) for (int i = tid; i < n2; i += kQpThreads) zs[i] = zg[i];
    else for (int i = tid; i < n2; i += kQpThreads) zg[i] = zs[i];
    __syncthreads();
    // (the polish left its own weights in the rows' per-solve fields; a factorisation would have rebuilt them)
    if (restore) rows_prepare_weights(q, sysw);
  };
  { PROF_T0(); factor_ok = factorize(sysw); PROF_ADD(6); }
#ifdef TB200_PROFILE
  sysw.prof_kind = 1;  // every later factorisation of the ADMM system: a rho update or the recovery after a failed polish
#endif

  double* dxs = q.scratch;              // [Np] last trajectory step (written on check iterations)
  double* dyb = q.scratch + q.Np;       // [Np] last dual step of the variable-bound rows
  double* st_x = q.scratch + 2 * q.Np;  // ADMM x, zb, yb stashed while polish reuses the shared vectors
  double* st_zb = q.scratch + 3 * q.Np;
  double* st_yb = q.scratch + 4 * q.Np;
  double pri_res = 0.0, dua_res = 0.0;
  int status = factor_ok ? QPS_UNSOLVED : QPS_NONCVX;
  bool early_verified = false;
  unsigned long long prev_guess = 0ull, failed_guess = 0ull, pending_guess = 0ull;
  bool have_prev_guess = false, have_failed_guess = false;
  double n_z = 0, n_ax = 0, n_q = 0, n_aty = 0, n_px = 0, s_pri = 0, s_dua = 0, s_z = 0, s_ax = 0, s_q = 0, s_aty = 0, s_px = 0;

  // ---------------------------------------------------------------- update_info(): residuals and norms
  // `scaled`: also the norms of the scaled quantities (only the rho estimate reads them)
  auto info_pass = [&](const bool scaled) {
    PROF_CHK_T0();
    p_matvec<NB>(q, q.x, q.v2);  // v2 <- P x
    PROF_CHK(4);
    double m[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    // 0 pri 1 z 2 ax 3 dua 4 aty 5 q 6 px | 7..13 the same on the scaled quantities
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      const double* R = q.R(r);
      double* F = q.F(r);
      const double ax = row_dot<CNc>(q, R, q.I(r), q.x) + F[R_U0] * F[R_XA0] + F[R_U1] * F[R_XA1];
      info_row_terms(F, ax, m);
      F[R_COEF] = F[R_Y];
    }
    __syncthreads();
    PROF_CHK(14);
    scatter_columns<CNc>(q, [&](int i) { return q.beta[i] * q.yb[i]; });  // v1 <- A'y (trajectory part)
    for (int i = tid; i < N; i += kQpThreads)
      info_var_terms(q.Dz[i], q.beta[i], q.x[i], q.zb[i], q.v1[i], q.v2[i], q.qs[i], m);
    if (scaled) {  // (block-uniform)
      block_reduce<14, 0u>(q, m);
      s_pri = m[7]; s_z = m[8]; s_ax = m[9]; s_dua = m[10]; s_aty = m[11]; s_q = m[12]; s_px = m[13];
    } else {
      double m7[7] = {m[0], m[1], m[2], m[3], m[4], m[5], m[6]};
      block_reduce<7, 0u>(q, m7);
#pragma unroll
      for (int k = 0; k < 7; ++k) m[k] = m7[k];
    }
    PROF_CHK(15);
    pri_res = m[0];
    dua_res = m[3] * q.cinv;
    n_z = m[1]; n_ax = m[2]; n_aty = m[4]; n_q = m[5]; n_px = m[6];
  };

  // The check fused into the last iteration of an ADMM block (admm_block_pinv, keep_last == 2): quantity k (ChkQ)
  // reduced from its warp partials in q.tmp, in the order of block_reduce.  Read where each quantity is needed (nothing
  // of it is carried across the ADMM loop); every writer of q.tmp is behind a barrier that follows these reads.
  auto fused_q = [&](const int k) -> double {
    extern __shared__ double sm[];
    const double* const chk = sm + (q.tmp - q.smbase) + k * 8;
    if ((kChkSumMask >> k) & 1u) {
      double acc = chk[0];
      for (int w = 1; w < kQpThreads / 32; ++w) acc += chk[w];
      return acc;
    }
    return warp_max_norm(chk[tid & 7]);
  };
  // the residuals of the current iterate: from the fused check when q.tmp holds it
  auto residuals = [&](const bool scaled) {
    if (!fused_chk) {
      info_pass(scaled);
      return;
    }
    double m[14];
#pragma unroll
    for (int k = 0; k < 14; ++k) m[k] = (k < 7 || scaled) ? fused_q(k) : 0.0;
    pri_res = m[0];
    dua_res = m[3] * q.cinv;
    n_z = m[1]; n_ax = m[2]; n_aty = m[4]; n_q = m[5]; n_px = m[6];
    if (scaled) { s_pri = m[7]; s_z = m[8]; s_ax = m[9]; s_dua = m[10]; s_aty = m[11]; s_q = m[12]; s_px = m[13]; }
  };

  auto primal_infeasible = [&](double eps) -> bool {  // is_primal_infeasible [EXT]
    double a[3] = {0.0, 0.0, 0.0};  // nd (max), lhs (sum), na (max)
    if (fused_chk) {
      a[0] = fused_q(CHK_PA0); a[1] = fused_q(CHK_PA1); a[2] = fused_q(CHK_PA2);
    } else {
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        double* F = q.F(r);
        F[R_COEF] = pinf_row_terms(F, q.I(r)[RI_AUX], a);  // projected dual step, consumed by the column pass
      }
      for (int i = tid; i < N; i += kQpThreads) pinf_var_terms(q.beta[i] / q.Dz[i], q.ubs[i], q.lbs[i], dyb[i], a);
      block_reduce<3, 0x2u>(q, a);
    }
    if (!((a[0] > eps) && (a[1] < -eps * a[0]))) return false;  // block-uniform: the A'dy test cannot rescue it
    if (fused_chk) {  // the projected dual steps for the column pass (the generic first stage leaves them in R_COEF)
      double unused[3] = {0.0, 0.0, 0.0};
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        double* F = q.F(r);
        F[R_COEF] = pinf_row_terms(F, q.I(r)[RI_AUX], unused);
      }
      __syncthreads();
    }
    scatter_columns<CNc>(q, [&](int i) { return q.beta[i] * dyb[i]; });
    double mm[1] = {a[2]};
    for (int i = tid; i < N; i += kQpThreads) mm[0] = fmax(mm[0], fabs(q.v1[i] / q.Dz[i]));
    block_reduce<1, 0u>(q, mm);
    return (a[0] > eps) && (a[1] < -eps * a[0]) && (mm[0] < eps * a[0]);
  };
  auto dual_infeasible = [&](double eps) -> bool {  // is_dual_infeasible [EXT]
    double a[2] = {0.0, 0.0};  // ndx (max), qdx (sum)
    if (fused_chk) {
      a[0] = fused_q(CHK_DA0); a[1] = fused_q(CHK_DA1);
    } else {
      for (int i = tid; i < N; i += kQpThreads) {
        a[0] = fmax(a[0], fabs(q.Dz[i] * dxs[i]));
        a[1] += q.qs[i] * dxs[i];
      }
      for (int r = tid; r < q.nrows; r += kQpThreads) dinf_row_terms(q.F(r), a);
      block_reduce<2, 0x2u>(q, a);
    }
    const double ndx = a[0], qdx = a[1];
    if (!((ndx > eps) && (qdx < -q.c * eps * ndx))) return false;  // block-uniform: skip the P dx / A dx tests
    for (int i = tid; i < q.Np; i += kQpThreads) q.v1[i] = (i < N) ? dxs[i] : 0.0;
    __syncthreads();
    p_matvec<NB>(q, q.v1, q.v2);  // v2 <- P dx
    double b2[2] = {0.0, 0.0};  // max |Dinv P dx|, bad count (sum)
    for (int i = tid; i < N; i += kQpThreads) {
      b2[0] = fmax(b2[0], fabs(q.v2[i] / q.Dz[i]));
      const double vv = q.Dz[i] * q.v1[i];  // Einv * (Eb Dz dx); both bounds finite
      b2[1] += (vv > eps * ndx || vv < -eps * ndx) ? 1.0 : 0.0;
    }
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      const double* R = q.R(r);
      const double* F = q.F(r);
      const int naux = q.I(r)[RI_AUX];
      const double ax = row_dot<CNc>(q, R, q.I(r), q.v1) + F[R_U0] * F[R_DXA0] + F[R_U1] * F[R_DXA1];
      const double vv = ax / F[R_E];
      b2[1] += (vv > eps * ndx) ? 1.0 : 0.0;                              // u finite for every row
      b2[1] += (naux != AUX_HINGE && vv < -eps * ndx) ? 1.0 : 0.0;        // l finite unless hinge
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const double va = F[R_B0 + k] * F[R_DXA0 + k] / F[R_EA0 + k];
        b2[1] += (k < naux && va < -eps * ndx) ? 1.0 : 0.0;               // aux rows: l = 0 finite, u infinite
      }
    }
    block_reduce<2, 0x2u>(q, b2);
    return (ndx > eps) && (qdx < -q.c * eps * ndx) && (b2[0] < q.c * eps * ndx) && (b2[1] == 0.0);
  };
  auto check_termination = [&](bool approximate) -> int {
    double eps_abs = st.eps_abs * eps_scale, eps_rel = st.eps_rel * eps_scale, epi = st.eps_prim_inf, edi = st.eps_dual_inf;
    if (approximate) {
      eps_abs *= 10; eps_rel *= 10; epi *= 10; edi *= 10;
    }
    const double eps_pri = eps_abs + eps_rel * fmax(n_z, n_ax);
    const double eps_dua = eps_abs + eps_rel * q.cinv * fmax(n_q, fmax(n_aty, n_px));
    const bool pri_ok = pri_res < eps_pri, dua_ok = dua_res < eps_dua;
    int res = QPS_UNSOLVED;
    if (pri_res > kOsqpInf || dua_res > kOsqpInf) res = QPS_NONCVX;
    else if (pri_ok && dua_ok) res = approximate ? QPS_SOLVED_INACC : QPS_SOLVED;
    else {  // block-uniform branch; the certificates are only evaluated when their residual test failed
      const bool pinf = pri_ok ? false : primal_infeasible(epi);
      const bool dinf = dua_ok ? false : dual_infeasible(edi);
      if (pinf) res = approximate ? QPS_PINF_INACC : QPS_PINF;
      else if (dinf) res = approximate ? QPS_DINF_INACC : QPS_DINF;
    }
    return res;
  };

  // ---------------------------------------------------------------- optimisation O1: when to try the polish early
  // The polish is tried early only when the hash of the active-set guess (guess_row_hash / guess_var_hash) is the same
  // as at the previous test and has not failed before.
  auto early_guess_settled = [&]() -> bool {
    unsigned long long h = 0ull;
    if (fused_chk) {
      extern __shared__ double sm[];
      const unsigned long long* hw = reinterpret_cast<const unsigned long long*>(sm + (q.tmp - q.smbase) + kChkHash * 8);
      for (int w = 0; w < kQpThreads / 32; ++w) h += hw[w];
    } else {
      for (int r = tid; r < q.nrows; r += kQpThreads) h += guess_row_hash(q.F(r), q.I(r), r, q.nrows, N);
      for (int i = tid; i < N; i += kQpThreads) h += guess_var_hash(q.zb[i], q.yb[i], q.lbs[i], q.ubs[i], i, q.nrows);
      // block sum (wraps): butterfly inside the warp, then the 8 partials through shared memory
      __syncwarp();
      for (int off = 16; off > 0; off >>= 1) h += __shfl_xor_sync(0xffffffffu, h, off);
      unsigned long long* red = reinterpret_cast<unsigned long long*>(q.red.ptr());
      if ((tid & 31) == 0) red[tid >> 5] = h;
      __syncthreads();
      h = 0ull;
      for (int w = 0; w < kQpThreads / 32; ++w) h += red[w];
      __syncthreads();
    }
    const bool stable = have_prev_guess && h == prev_guess;
    prev_guess = h;
    have_prev_guess = true;
    pending_guess = h;
    return stable && !(have_failed_guess && h == failed_guess);
  };

  // ADMM iterations, continuing from the current state until a termination test fires or max_iter is reached.
  auto run_admm = [&](auto& polish_fn, auto& restore_fn) {
    status = QPS_UNSOLVED;
    bool stop = false;
    while (!stop) {
      if (iter >= st.max_iter) {  // max_iter reached without a verdict: approximate test, then MAX_ITER_REACHED
        if (!(st.check_termination > 0 && (iter % st.check_termination == 0))) residuals(false);
        status = check_termination(true);
        if (status == QPS_UNSOLVED) status = QPS_MAXITER;
        stop = true;
      } else {
        // the iterations up to the next event (termination test, rho update, max_iter) run as one block
        int n = st.max_iter - iter;
        if (st.check_termination > 0) n = min(n, st.check_termination - iter % st.check_termination);
        if (st.adaptive_rho && st.adaptive_rho_interval > 0) n = min(n, st.adaptive_rho_interval - iter % st.adaptive_rho_interval);
        iter += n;
        const bool can_check = st.check_termination > 0 && (iter % st.check_termination == 0);
        const bool rho_iter = st.adaptive_rho && st.adaptive_rho_interval > 0 && (iter % st.adaptive_rho_interval == 0);
        run_block(n, can_check || iter == st.max_iter);
        if (can_check) {
          PROF_T0();
          residuals(rho_iter);
          PROF_CHK_T0();
          status = check_termination(false);
          PROF_CHK(9);
          PROF_ADD(5);
          bool try_early = false;
          if (status != QPS_UNSOLVED) stop = true;
          else if (st.polishing && st.early_polish_every > 0 && iter >= st.early_polish_from &&
                   (iter % st.early_polish_every == 0)) {
            PROF_T0();
            try_early = early_guess_settled();
            PROF_ADD(22);
          }
          if (try_early) {
            // optimisation O1: try the polish before ADMM has met its own tolerances; a VERIFIED polished point
            // is the exact minimiser no matter how rough the iterate that produced the active-set guess was
            bool verified = false;
            double p_pri = 0.0, p_dua = 0.0;
            PROF_COUNT(17);
            { PROF_T0(); if (use_pinv) stash_z(false); PROF_ADD(16); }
            const bool factored = polish_fn(verified, p_pri, p_dua);
            if (factored && verified) {
              early_verified = true;
              out.pol_factor_ok = 1;
              out.pol_pri = p_pri;
              out.pol_dua = p_dua;
              status = QPS_SOLVED;
              stop = true;
            } else {
              PROF_T0();
              failed_guess = pending_guess;
              have_failed_guess = true;
              // x, zb, yb come back exactly and the polish writes none of the row fields the residual norms read, so
              // the residual scalars of this check (pri_res, dua_res, n_*, s_*) still hold: no second info_pass.  (It
              // does overwrite R_COEF and, through its factorisation, q.tmp: a certificate evaluated after this point
              // takes the generic first stage, which rebuilds both from the iterate.)
              restore_fn(false);
              if (use_pinv) {
                stash_z(true);
              } else if (!factorize(sysw)) {
                status = QPS_NONCVX;
                stop = true;
              }
              PROF_ADD(19);
            }
          }
        }
        if (!stop && rho_iter) {
          if (!can_check) residuals(true);
          // compute_rho_estimate on the scaled quantities [EXT]
          const double pn = s_pri / (fmax(s_z, s_ax) + 1e-10);
          const double dn = s_dua / (fmax(s_q, fmax(s_aty, s_px)) + 1e-10);
          double rho_new = rho * sqrt(pn / (dn + 1e-10));
          rho_new = fmin(fmax(rho_new, kRhoMin), kRhoMax);
          if (rho_new > rho * st.adaptive_rho_tolerance || rho_new < rho / st.adaptive_rho_tolerance) {
            rho = rho_new;
            q.rho = rho;
            q.rho_eq = kRhoEqOverIneq * rho;
            sysw.rho_aux = rho;
            out.rho_updates++;
            PROF_T0();
            if (!factorize(sysw)) {
              status = QPS_NONCVX;
              stop = true;
            }
            PROF_ADD(20);
          }
        }
      }
    }
  };

  // ---------------------------------------------------------------- polish (OSQP polish.c [EXT])
  // Equality-constrained QP on the guessed active set, solved as the delta-regularised KKT system with
  // iterative refinement, in its reduced form K_p = P + delta I + (1/delta) A_act' A_act (same aux
  // elimination and block factor as the ADMM system).  Returns false when K_p could not be factored.
  // `verified`: the polished point is primal feasible to kVerifyTol and every active inequality row has a
  // correctly signed multiplier, i.e. it is a KKT point of the QP = the unique minimiser.
  const double wp = 1.0 / st.delta;
  const SysW pw{true, st.delta, 0.0};
  // the refinement passes on the factored polish system
  auto polish_refine = [&](bool& verified, double& p_pri, double& p_dua) {
    PROF_T0();
    if constexpr (REGOK) {
      if (fast_polish) {
        using PassFn = PolishRes (*)(const QpCtx&, int);
        PassFn volatile fn = &polish_passes<NB, PAIR>;
        const PolishRes res = fn(q, st.polish_refine_iter);
        p_pri = res.p_pri;
        p_dua = res.p_dua;
        verified = (res.bad == 0.0) && (p_pri <= kVerifyTol) && isfinite(p_pri) && isfinite(p_dua);
        PROF_ADD(12);
        return;
      }
    }
    for (int it = 0; it <= st.polish_refine_iter + 1; ++it) {
      const bool last = (it == st.polish_refine_iter + 1);  // final pass: pending dual update + residuals only
      p_matvec<NB>(q, q.x, q.v2);  // v2 <- P xq
      double mm[3] = {0.0, 0.0, 0.0};  // m_pri (max), m_dua (max), bad signs (sum)
      // rows: residual of the row, pending multiplier update, aux right-hand sides, row multiplier for A'
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        const double* R = q.R(r);
        double* F = q.F(r);
        const int naux = q.I(r)[RI_AUX];
        const double Wr = F[R_WRR];
        const double ax = row_dot<CNc>(q, R, q.I(r), q.x) + F[R_U0] * F[R_PX0] + F[R_U1] * F[R_PX1];
        const double py = F[R_PY] + ((it > 0) ? Wr * (ax - F[R_PB]) : 0.0);
        const double e = py + (last ? 0.0 : Wr * (ax - F[R_PB]));
        const double zc = fmin(fmax(ax, F[R_LO]), F[R_UP]);
        mm[0] = fmax(mm[0], fabs((ax - zc) / F[R_E]));
        mm[2] += (last && Wr != 0.0 && naux == AUX_HINGE && py < -kVerifyTol) ? 1.0 : 0.0;  // upper active needs y >= 0
        double pya[2], ra[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const double bb = F[R_B0 + k], u = F[R_U0 + k], qa = F[R_QA0 + k];
          const double wa = fabs(F[R_PWA0 + k]);
          const double axb = bb * F[R_PX0 + k];
          pya[k] = F[R_PYA0 + k] + ((it > 0) ? wa * axb : 0.0);
          const double ea = pya[k] + (last ? 0.0 : wa * axb);
          mm[0] = fmax(mm[0], fabs((axb - fmax(axb, 0.0)) / F[R_EA0 + k]));
          mm[2] += (last && wa != 0.0 && pya[k] > kVerifyTol) ? 1.0 : 0.0;  // aux >= 0 held at 0 needs y <= 0
          mm[1] = fmax(mm[1], fabs((qa + u * py + bb * pya[k]) / F[R_DA0 + k]));
          ra[k] = -qa - u * e - bb * ea;
        }
        F[R_PY] = py;
        F[R_PYA0] = pya[0];
        F[R_PYA1] = pya[1];
        F[R_RA0] = ra[0];
        F[R_RA1] = ra[1];
        F[R_COEF] = last ? py : row_reduce_coef(F, ra[0], ra[1], -e);
      }
      __syncthreads();
      if (last) {
        // dual residual  P x + q + A'y  over the trajectory variables
        scatter_columns<CNc>(q, [&](int i) { return q.v2[i] + q.qs[i] + q.beta[i] * q.yb[i]; });
      } else {
        // rd = -(P x + q) - beta * (y + W (A x - b)) + A' coef
        scatter_columns<CNc>(q, [&](int i) {
          const double beta = q.beta[i];
          const double w = fabs(q.zb[i]);
          const double bnd = q.zb[i] > 0 ? q.ubs[i] : q.lbs[i];
          return -(q.v2[i] + q.qs[i]) - beta * (q.yb[i] + w * (beta * q.x[i] - bnd));
        });
      }
      for (int i = tid; i < N; i += kQpThreads) {
        const double beta = q.beta[i];
        const double ax = beta * q.x[i];
        const double w = fabs(q.zb[i]);
        const double lb = q.lbs[i], ub = q.ubs[i];
        const double zc = fmin(fmax(ax, lb), ub);
        mm[0] = fmax(mm[0], fabs((ax - zc) * q.Dz[i] / beta));
        const bool ineq = last && w != 0.0 && (ub - lb >= kRhoTol);
        mm[2] += (ineq && q.zb[i] > 0 && q.yb[i] < -kVerifyTol) ? 1.0 : 0.0;
        mm[2] += (ineq && q.zb[i] < 0 && q.yb[i] > kVerifyTol) ? 1.0 : 0.0;
        if (last) mm[1] = fmax(mm[1], fabs(q.v1[i] / q.Dz[i]));
      }
      if (last) {
        block_reduce<3, 0x4u>(q, mm);
        p_pri = mm[0];
        p_dua = mm[1] * q.cinv;
        verified = (mm[2] == 0.0) && (p_pri <= kVerifyTol) && isfinite(p_pri) && isfinite(p_dua);
      } else {
        bcr_solve<NB>(q, q.v1, q.w);  // (five solves per polish: factor rows read from memory)
        for (int r = tid; r < q.nrows; r += kQpThreads) {
          const double* R = q.R(r);
          double* F = q.F(r);
          double a0, a1;
          row_backsub(F, row_dot<CNc>(q, R, q.I(r), q.w), a0, a1);
          F[R_PX0] += a0;
          F[R_PX1] += a1;
        }
        for (int i = tid; i < N; i += kQpThreads) {
          const double xn = q.x[i] + q.w[i];
          // multiplier update of the variable-bound rows with the new iterate (the rows do theirs at the
          // start of the next pass, where A x is recomputed anyway)
          const double w = fabs(q.zb[i]);
          q.yb[i] += w * (q.beta[i] * xn - (q.zb[i] > 0 ? q.ubs[i] : q.lbs[i]));
          q.x[i] = xn;
        }
        __syncthreads();
      }
    }
    PROF_ADD(12);
  };
  auto polish_once = [&](bool& verified, double& p_pri, double& p_dua) -> bool {
    PROF_COUNT(13);
    PROF_T0();
    verified = false;
    for (int i = tid; i < q.Np; i += kQpThreads) {
      const double z = q.zb[i], y = q.yb[i];
      double w = 0.0;
      if (i < N) {
        if (z - q.lbs[i] < -y) w = -wp;           // lower active
        else if (q.ubs[i] - z < y) w = wp;        // upper active
      }
      st_x[i] = q.x[i];
      st_zb[i] = z;
      st_yb[i] = y;
      q.zb[i] = w;                                 // signed polish weight
      q.x[i] = 0.0;                                // polish iterate
      q.yb[i] = 0.0;                               // polish multiplier
    }
    for (int r = tid; r < q.nrows; r += kQpThreads) {
      double* F = q.F(r);
      const int naux = q.I(r)[RI_AUX];
      double w = 0.0, b = 0.0;
      if (F[R_Z] - F[R_LO] < -F[R_Y]) { w = -wp; b = F[R_LO]; }
      else if (F[R_UP] - F[R_Z] < F[R_Y]) { w = wp; b = F[R_UP]; }
      F[R_PW] = w;
      F[R_PB] = b;
      F[R_PY] = 0.0;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        double wa = 0.0;
        if (k < naux) {
          if (F[R_ZA0 + k] - 0.0 < -F[R_YA0 + k]) wa = -wp;                                    // lower (0) active
          else if (kOsqpInf * F[R_EA0 + k] - F[R_ZA0 + k] < F[R_YA0 + k]) wa = wp;            // never in practice
        }
        F[R_PWA0 + k] = wa;
        F[R_PYA0 + k] = 0.0;
        F[R_PX0 + k] = 0.0;
      }
    }
    __syncthreads();
    PROF_ADD(16);
    bool factored;
    { PROF_T0(); factored = factorize(pw); PROF_ADD(23); }
    if (!factored) return false;
    polish_refine(verified, p_pri, p_dua);
    return true;
  };
  auto restore_admm_state = [&](bool keep_polished_x) {
    for (int i = tid; i < q.Np; i += kQpThreads) {
      if (!keep_polished_x) q.x[i] = st_x[i];
      q.zb[i] = st_zb[i];
      q.yb[i] = st_yb[i];
    }
    __syncthreads();
  };

  // ---- main loop: ADMM -> polish -> verify; on a failed verification ADMM continues with 10x tighter ------
  // tolerances (DESIGN.md deviation D2).
  bool done = !factor_ok;
  while (!done) {
    run_admm(polish_once, restore_admm_state);
    out.pri_res = pri_res;
    out.dua_res = dua_res;
    if (status != QPS_SOLVED || !st.polishing) {
      done = true;
    } else if (early_verified) {
      out.polish = 1;
      out.rounds = round;
      done = true;
    } else {
      bool verified = false;
      double p_pri = 0.0, p_dua = 0.0;
      PROF_COUNT(18);
      { PROF_T0(); if (use_pinv) stash_z(false); PROF_ADD(16); }
      const bool factored = polish_once(verified, p_pri, p_dua);
      out.pol_factor_ok = factored ? 1 : 0;
      out.pol_pri = p_pri;
      out.pol_dua = p_dua;
      out.rounds = round;
      if (factored && verified) {
        out.polish = 1;
        done = true;
      } else if (round >= kVerifyRounds || iter >= st.max_iter) {  // OSQP's acceptance rule
        const bool ok = factored && ((p_pri < pri_res && p_dua < dua_res) || (p_pri < pri_res && dua_res < 1e-10) ||
                                     (p_dua < dua_res && pri_res < 1e-10)) && isfinite(p_pri) && isfinite(p_dua);
        out.polish = ok ? 2 : -1;
        done = true;
      } else {
        ++round;
        eps_scale *= 0.1;
        PROF_T0();
        restore_admm_state(false);
        if (use_pinv) {  // back to the ADMM factor
          stash_z(true);
        } else if (!factorize(sysw)) {
          status = QPS_NONCVX;
          done = true;
        }
        PROF_ADD(19);
      }
    }
  }
  out.iters = iter;
  out.status = status;
  out.rho = rho;
  out.c = q.c;
  if (out.polish != 0) {
    // Adopt the polished PRIMAL point when accepted.  The duals kept for the next warm start are always the
    // ADMM duals: polished duals are non-unique on degenerate active sets (DESIGN.md deviation D1).
    if (out.polish > 0) {
      for (int r = tid; r < q.nrows; r += kQpThreads) {
        double* F = q.F(r);
        for (int k = 0; k < 2; ++k) F[R_XA0 + k] = F[R_PX0 + k];
      }
    }
    restore_admm_state(out.polish > 0);
  }
  return out;
}

// ---------------------------------------------------------------------------------------------------
// QP assembly (optimizers.cpp:781-799 + osqp_interface.cpp:170-281 in fixed layout) + solve of trajectory b by the
// calling CTA (256 threads).  DD = degrees of freedom (block size NB = 2*DD); PAIR: rows may span two waypoints.
// The row of an AvoidSingularity object (problem_description.cpp:1900-1939): 1 row over q_first, D coefficients; an ABS
// cost row or an INEQ constraint row (hinge), the coefficients with |g| <= 1e-7 of the unscaled gradient dropped
// (cleanupAff, modeling_utils.cpp:143-211, 238-269).  Written by thread 0; returns the row's entries of A (its real
// coefficients and aux columns).  Called only by the SING instances of qp_step.
static __device__ __noinline__ int qp_singularity_row(const DevProblem& p, const QpCtx& q, const DevObj& o, const int oi,
                                                      const bool is_cnt, const double w_aux, const double* cart_err,
                                                      const double* cart_jac, const int nr, const int n_aux, int* sh_i) {
  const int D = q.D;
  if (q.tid == 0) {
    double* R = q.R(nr);
    int* I = q.rints + static_cast<size_t>(nr) * RI_NINTS;
    const double* J = cart_jac + static_cast<size_t>(o.src_off) * p.cart_stride;
    const double thr = 1e-7 * fabs(o.coeff);
    double dot = 0.0;
    int nz = 0;
    for (int j = 0; j < q.CN; ++j) {
      const double Jj = (j < D) ? J[j] : 0.0;
      dot += Jj * q.x[o.first * D + min(j, D - 1)];
      const double a = (fabs(Jj) > thr) ? Jj : 0.0;
      R[j] = a;
      nz += (a != 0.0);
    }
    R[2 * q.CN + R_C] = cart_err[o.src_off] - dot;
    R[2 * q.CN + R_W] = w_aux;
    I[RI_BASE] = o.first * D; I[RI_CNT] = D; I[RI_STRIDE] = 1; I[RI_AUX] = is_cnt ? AUX_HINGE : AUX_ABS;
    I[RI_OBJ] = oi; I[RI_PAD] = n_aux;
    sh_i[0] = nz;
  }
  __syncthreads();
  const int nz = sh_i[0];
  __syncthreads();
  return nz + (is_cnt ? 1 : 2);
}

// SING: the instance for problems with AvoidSingularity objects (the row builder of SING = 0 has no branch for them)
template <int DD, int PAIR, int SING = 0>
__device__ __noinline__ void qp_step(const DevProblem& p, const int b, const double* x_override /*kernel-level API*/,
                                        const double* trust_override, int* admm_iters_out, int* polish_out) {
  constexpr int NB = 2 * DD;
  constexpr bool FG = DD > 8;  // blocks of more than 16: the factor lives in this CTA's region of global memory
  extern __shared__ double sm[];
  const int tid = threadIdx.x;
  if (!x_override && (p.status[b] != 5 || p.qp_done[b] != 0)) return;  // finished, or waiting for its evaluation
  const int N = p.N, T = p.T, D = p.D;
  QpCtx q;
  q.N = N; q.T = T; q.D = D; q.tid = tid;
  q.nb = NB;
  q.M = qp_block_count(N, NB);
  q.Np = q.M * NB;
  q.CN = (p.row_stride - R_NF) / 3;
  q.RS = p.row_stride;
  const QpSmem S = qp_smem_layout(N, NB, q.RS, q.CN, p.max_rows, FG);
  if (FG || !S.factor_smem) {  // (a factor of <= 16-wide blocks that does not fit shared memory goes the same way)
    double* fg = p.factor_g + static_cast<size_t>(blockIdx.x) * qp_cta_global_doubles(N, NB);
    const int fb = qp_even(q.M * NB * NB);
    q.SA = fg; q.SLM = fg + fb; q.SU = fg + 2 * fb;
  } else {
    q.SA = sm + S.SA; q.SLM = sm + S.SLM; q.SU = sm + S.SU;
  }
  q.beta = sm + S.beta;
  q.x = sm + S.x; q.zb = sm + S.zb; q.yb = sm + S.yb; q.v1 = sm + S.v1; q.w = sm + S.w;
  q.qs = sm + S.qs; q.lbs = sm + S.lbs; q.ubs = sm + S.ubs; q.tmp = sm + S.tmp; q.red = sm + S.red;
  q.flag = sm + S.red - 8;
  q.colptr = reinterpret_cast<int*>(sm + S.colptr);
  double* const rows_g = p.rows + static_cast<size_t>(b) * p.max_rows * p.row_stride;
  int* const rints_g = p.row_ints + static_cast<size_t>(b) * p.max_rows * RI_NINTS;
  q.rows = rows_g;
  q.soa = p.soa + static_cast<size_t>(blockIdx.x) * p.soa_stride;
  q.smbase = sm;
  q.pinv = S.pinv;
  q.pl = pinv_plan(q.M, NB);
  q.pi_g = p.factor_g + static_cast<size_t>(blockIdx.x) * qp_cta_global_doubles(N, NB);
  q.z_stash = q.pi_g + qp_factor_doubles(N, NB);
  q.rows_smem = 0;
  q.rints = rints_g;
  int* mylist = p.lists + static_cast<size_t>(b) * p.list_stride;
  int* colptr = mylist;                                   // [Np+1] master copy (shared copy in q.colptr)
  int* colent = mylist + q.Np + 1;                        // [max_rows*CN]
  int* obj_start = colent + static_cast<size_t>(p.max_rows) * q.CN;  // [n_objs+1]
  q.colent = colent;
  q.band_offs = p.band_offs;
  q.n_band = p.n_band;
  if (S.pband_smem) {
    q.Pband = sm + S.Pb;
    for (int t = tid; t < N * (NB + 1); t += kQpThreads) sm[S.Pb + t] = p.Pband[t];
  } else {
    q.Pband = p.Pband;  // long trajectories: the band stays in (L2-resident) global memory
  }
  // per-trajectory global vectors: dxs dyb st_x st_zb st_yb (the ADMM state stashed while the polish runs)
  double* gvec = p.scratch + static_cast<size_t>(b) * 5 * q.Np;
  q.scratch = gvec;
  q.Dz = sm + S.Dz;
  q.v2 = sm + S.v2;
  double *qs = q.qs, *lbs = q.lbs, *ubs = q.ubs;
  int* meta = p.ws_meta + static_cast<size_t>(b) * 8;  // 0..3 warm-start key (n_aux, rows, nnzA, last status)
  const int n_obj = p.n_costs + p.n_cnts;
  int nr = 0, n_aux = 0, nnzA = 0;
  bool warm = false;
  int* sh_i = reinterpret_cast<int*>(q.flag + 2);  // small shared int scratch during assembly

  {
    const double* xc = (x_override ? x_override : p.x) + static_cast<size_t>(b) * N;
    const double trust = trust_override ? trust_override[b] : p.trust[b];
    const double* mu = p.merit_coeffs + static_cast<size_t>(b) * p.n_cnts;
    const int buf = x_override ? 0 : p.cur_buf[b];
    const size_t slot = static_cast<size_t>(buf) * p.B + b;
    const double* cart_err = p.cart_err + slot * p.n_cart_rows;
    const double* cart_jac = p.cart_jac + slot * static_cast<size_t>(p.n_cart_rows) * p.cart_stride;
    const double* coll_rows = p.coll_rows + slot * static_cast<size_t>(p.n_coll_cand) * p.coll_stride;
    const unsigned long long* coll_mask = p.coll_mask + slot * static_cast<size_t>(p.n_coll_objs) * p.coll_words;

    // ---- trajectory part: x, trust box (setTrustBoxConstraints, optimizers.cpp:151-170), linear cost -----
    for (int i = tid; i < N; i += kQpThreads) {
      const double lb = p.lower[i % D], ub = p.upper[i % D];
      const double xi = fmin(fmax(xc[i], lb), ub);
      lbs[i] = fmax(fmax(xi - trust, lb), -kOsqpInf);
      ubs[i] = fmin(fmin(xi + trust, ub), kOsqpInf);
      qs[i] = p.qlin[i];
      q.x[i] = xc[i];  // linearisation point (until the solver takes over x)
    }
    __syncthreads();

    // ---- rows in the reference's canonical order: permanent rows, cost rows, penalised constraint rows -----
    // (every record is padded: CN coefficients, zeros beyond the row's own count)
    for (int f = tid; f < p.n_fixed; f += kQpThreads) {  // fixed_timesteps / fixed_dofs rows: x_k - init_k == 0
      const int var = p.fixed_vars[f];
      double* R = q.R(f);
      int* I = q.rints + static_cast<size_t>(f) * RI_NINTS;
      for (int k = 0; k < q.CN; ++k) R[k] = (k == 0) ? 1.0 : 0.0;
      R[2 * q.CN + R_C] = -p.init_traj[static_cast<size_t>(b) * N + var];
      R[2 * q.CN + R_W] = 0.0;
      I[RI_BASE] = var; I[RI_CNT] = 1; I[RI_STRIDE] = D; I[RI_AUX] = AUX_NONE; I[RI_OBJ] = -1; I[RI_PAD] = 0;
    }
    nr += p.n_fixed;
    nnzA += p.n_fixed;
    int coll_obj_counter = 0;
    for (int oi = 0; oi < n_obj; ++oi) {
      const bool is_cnt = oi >= p.n_costs;
      const DevObj o = is_cnt ? p.cnt_objs[oi - p.n_costs] : p.cost_objs[oi];
      if (tid == 0) obj_start[oi] = nr;
      const double w_aux = is_cnt ? mu[oi - p.n_costs] : 1.0;
      if (o.kind == OBJ_JOINT_EQ_COST) continue;
      if (o.kind == OBJ_JOINT_EQ_CNT || o.kind == OBJ_JOINT_INEQ_CNT || o.kind == OBJ_JOINT_INEQ_COST) {
        const DevJointTerm& jt = p.joint_terms[o.term];
        const int per = (o.kind == OBJ_JOINT_EQ_CNT) ? 1 : 2;
        const int total = o.n_steps * D * per;
        const double wst[3][3] = {{1, 0, 0}, {-1, 1, 0}, {1, -2, 1}};
        for (int k = tid; k < total; k += kQpThreads) {
          const int t = o.first + k / (D * per), d = (k / per) % D, side = k % per;
          double* R = q.R(nr + k);
          int* I = q.rints + static_cast<size_t>(nr + k) * RI_NINTS;
          const double cd = jt.coeffs[d];
          double sgn = cd, cst;
          if (per == 1) cst = -jt.targets[d] * cd;
          else if (side == 0) cst = (-jt.targets[d] - jt.upper[d]) * cd;        // (e - upper) * c
          else { sgn = -cd; cst = (jt.lower[d] + jt.targets[d]) * cd; }         // (lower - e) * c
          for (int i = 0; i < q.CN; ++i) R[i] = (i <= o.order) ? wst[o.order][i] * sgn : 0.0;
          R[2 * q.CN + R_C] = cst;
          R[2 * q.CN + R_W] = w_aux;
          I[RI_BASE] = t * D + d; I[RI_CNT] = o.order + 1; I[RI_STRIDE] = D;
          I[RI_AUX] = (per == 1) ? AUX_ABS : AUX_HINGE; I[RI_OBJ] = oi;
          I[RI_PAD] = n_aux + k * ((per == 1) ? 2 : 1);  // index of the row's first aux variable
        }
        nr += total;
        n_aux += total * ((per == 1) ? 2 : 1);
        nnzA += total * (o.order + 1 + ((per == 1) ? 2 : 1));
      } else if (o.kind == OBJ_CART_POSE) {
        const DevCartTerm& ct = p.cart_terms[o.term];
        if (tid == 0) sh_i[0] = 0;
        __syncthreads();
        int nz = 0;
        for (int k = tid; k < o.n_rows; k += kQpThreads) {
          double* R = q.R(nr + k);
          int* I = q.rints + static_cast<size_t>(nr + k) * RI_NINTS;
          const double* J = cart_jac + static_cast<size_t>(o.src_off + k) * p.cart_stride;
          const double thr = 1e-7 * fabs(ct.coeff[k]);  // cleanupAff acts on the unscaled gradient (modeling_utils.cpp:31-39)
          double dot = 0.0;
          for (int j = 0; j < q.CN; ++j) {
            const double Jj = (j < D) ? J[j] : 0.0;
            dot += Jj * q.x[o.first * D + min(j, D - 1)];
            const double a = (fabs(Jj) > thr) ? Jj : 0.0;
            R[j] = a;
            nz += (a != 0.0);
          }
          R[2 * q.CN + R_C] = cart_err[o.src_off + k] - dot;
          R[2 * q.CN + R_W] = w_aux;
          I[RI_BASE] = o.first * D; I[RI_CNT] = D; I[RI_STRIDE] = 1; I[RI_AUX] = AUX_ABS; I[RI_OBJ] = oi;
          I[RI_PAD] = n_aux + 2 * k;
        }
        if (nz) atomicAdd(&sh_i[0], nz);
        __syncthreads();
        nz = sh_i[0];
        __syncthreads();
        nr += o.n_rows;
        n_aux += 2 * o.n_rows;
        nnzA += nz + 2 * o.n_rows;
      } else if (o.kind == OBJ_CART_VEL) {
        // CartVel step pair: 6 rows over (q_t, q_t+1); INEQ constraint rows (hinge) or ABS cost rows
        // (problem_description.cpp:1011-1057, modeling_utils.cpp:143-211, 238-269; coefficients |c| <= 1e-7 dropped)
        if (tid == 0) sh_i[0] = 0;
        __syncthreads();
        int nz = 0;
        const int per = is_cnt ? 1 : 2;
        for (int k = tid; k < 6; k += kQpThreads) {
          double* R = q.R(nr + k);
          int* I = q.rints + static_cast<size_t>(nr + k) * RI_NINTS;
          const double* J = cart_jac + static_cast<size_t>(o.src_off + k) * p.cart_stride;
          double dot = 0.0;
          for (int j = 0; j < q.CN; ++j) {
            const double Jj = (j < 2 * D) ? J[j] : 0.0;
            dot += Jj * q.x[o.first * D + min(j, 2 * D - 1)];
            const double a = (fabs(Jj) > 1e-7) ? Jj : 0.0;
            R[j] = a;
            nz += (a != 0.0);
          }
          R[2 * q.CN + R_C] = cart_err[o.src_off + k] - dot;
          R[2 * q.CN + R_W] = w_aux;
          I[RI_BASE] = o.first * D; I[RI_CNT] = 2 * D; I[RI_STRIDE] = 1; I[RI_AUX] = is_cnt ? AUX_HINGE : AUX_ABS;
          I[RI_OBJ] = oi; I[RI_PAD] = n_aux + per * k;
        }
        if (nz) atomicAdd(&sh_i[0], nz);
        __syncthreads();
        nz = sh_i[0];
        __syncthreads();
        nr += 6;
        n_aux += per * 6;
        nnzA += nz + per * 6;
      } else if (SING != 0 && o.kind == OBJ_SINGULARITY) {
        nnzA += qp_singularity_row(p, q, o, oi, is_cnt, w_aux, cart_err, cart_jac, nr, n_aux, sh_i);
        nr += 1;
        n_aux += is_cnt ? 1 : 2;
      } else if (o.kind == OBJ_COLL || o.kind == OBJ_COLL_CAST) {
        // active candidates of this timestep, in candidate order: thread 0 scans the mask and assigns slots
        const unsigned long long* mw = coll_mask + static_cast<size_t>(coll_obj_counter) * p.coll_words;
        ++coll_obj_counter;
        // slot of candidate c = number of active candidates before it (popcount of the mask prefix)
        if (tid == 0) { sh_i[0] = 0; sh_i[1] = 0; }
        __syncthreads();
        int nz = 0;
        for (int c = tid; c < o.n_rows; c += kQpThreads) {
          const bool act = (mw[c / 64] >> (c % 64)) & 1ull;
          if (act) {
            int before = 0;
            for (int wdx = 0; wdx < c / 64; ++wdx) before += __popcll(mw[wdx]);
            before += __popcll(mw[c / 64] & ((1ull << (c % 64)) - 1ull));
            const int pos = nr + before;
            double* R = q.R(pos);
            int* I = q.rints + static_cast<size_t>(pos) * RI_NINTS;
            const double* cr = coll_rows + static_cast<size_t>(o.src_off + c) * p.coll_stride;
            // dist(q) ~ d0 + g.(q - q0);  constraint: coeff*(margin - dist) <= 0;  cost: hinge(margin - dist)*coeff
            // W coefficients: D (one waypoint) or 2*D (step pair of the continuous evaluator, where cleanupAff drops
            // |g| <= 1e-7: collision_terms.cpp:481,502,536)
            const int W = (o.kind == OBJ_COLL_CAST) ? 2 * D : D;
            const double thr = (o.kind == OBJ_COLL_CAST) ? 1e-7 : -1.0;
            const double scale = is_cnt ? cr[W + 2] : 1.0;
            double dot = 0.0;
            for (int j = 0; j < q.CN; ++j) {
              const double g = (j < W) ? cr[j] : 0.0;
              dot += g * q.x[o.first * D + min(j, W - 1)];
              const double a = (fabs(g) > thr) ? -g * scale : 0.0;
              R[j] = (j < W) ? a : 0.0;
              nz += (j < W && a != 0.0);
            }
            R[2 * q.CN + R_C] = (cr[W + 1] - cr[W] + dot) * scale;
            R[2 * q.CN + R_W] = is_cnt ? w_aux : cr[W + 2];
            I[RI_BASE] = o.first * D; I[RI_CNT] = W; I[RI_STRIDE] = 1; I[RI_AUX] = AUX_HINGE; I[RI_OBJ] = oi;
            I[RI_PAD] = n_aux + before;
          }
        }
        if (nz) atomicAdd(&sh_i[0], nz);
        __syncthreads();
        nz = sh_i[0];
        int count = 0;
        for (int wdx = 0; wdx < p.coll_words; ++wdx) count += __popcll(mw[wdx]);
        __syncthreads();
        nr += count;
        n_aux += count;
        nnzA += nz + count;
      }
    }
    if (tid == 0) obj_start[n_obj] = nr;
    nnzA += N + n_aux;  // identity rows carrying the variable bounds
    __syncthreads();

    // ---- per-column entry lists (canonical row order inside every column; real coefficients only) ---------
    for (int i = tid; i <= q.Np; i += kQpThreads) colptr[i] = 0;
    __syncthreads();
    for (int r = tid; r < nr; r += kQpThreads) {
      const int* I = q.I(r);
      for (int k = 0; k < I[RI_CNT]; ++k) atomicAdd(&colptr[I[RI_BASE] + k * I[RI_STRIDE] + 1], 1);
    }
    __syncthreads();
    if (tid == 0)
      for (int i = 0; i < q.Np; ++i) colptr[i + 1] += colptr[i];
    __syncthreads();
    // one thread per column walks the rows in canonical order (columns are short; rows are few)
    for (int i = tid; i < N; i += kQpThreads) {
      if (colptr[i + 1] == colptr[i]) continue;
      int pos = colptr[i];
      for (int r = 0; r < nr && pos < colptr[i + 1]; ++r) {
        const int* I = q.I(r);
        const int base = I[RI_BASE], stride = I[RI_STRIDE], cnt = I[RI_CNT];
        const int off = i - base;
        if (off >= 0 && off % stride == 0 && off / stride < cnt) colent[pos++] = (r << 5) | (off / stride);
      }
    }
    __syncthreads();
    q.nrows = nr;
  }
  for (int i = tid; i <= q.Np; i += kQpThreads) q.colptr[i] = colptr[i];
  __syncthreads();
  // ---- the rows move into shared memory when they fit (the common case) ---------------------------------
  const bool rows_in_smem = nr <= S.row_cap;
  double* const rows_s = sm + S.rows;
  if (rows_in_smem) {
    int* rints_s = reinterpret_cast<int*>(sm + S.rints);
    int* colent_s = reinterpret_cast<int*>(sm + S.colent);
    for (int t = tid; t < nr * q.RS; t += kQpThreads) rows_s[t] = rows_g[t];
    for (int t = tid; t < nr * RI_NINTS; t += kQpThreads) rints_s[t] = rints_g[t];
    for (int t = tid; t < q.colptr[q.Np]; t += kQpThreads) colent_s[t] = colent[t];
    q.rows = rows_s;
    q.rows_smem = 1;
    q.rints = rints_s;
    q.colent = colent_s;
  }
  __syncthreads();

  // ---- warm start decision (createOrUpdateSolver, osqp_interface.cpp:283-370) ---------------------------
  warm = !x_override && p.qp.warm_starting && meta[3] == 1 && meta[0] == n_aux && meta[1] == nr && meta[2] == nnzA;
  { PROF_T0(); qp_scale(q, p.qp, n_aux); PROF_ADD(7); }
  __syncthreads();

  PROF_T0();
  QpOut res = qp_solve_block<NB, PAIR, (DD <= 7)>(q, p.qp, warm, p.ws_rho[b], p.ws_x + static_cast<size_t>(b) * N,
                                                  p.ws_yb + static_cast<size_t>(b) * N, p.qp_fast_passes != 0);
  __syncthreads();
  PROF_ADD(8);
#ifdef TB200_PROFILE
  if (tid == 0) atomicAdd(&g_prof[9], 1ull);
#endif

  // ---- unscale, store the solution (and the warm-start state), model values -----------------------------
  double* nx = p.new_x + static_cast<size_t>(b) * N;
  for (int i = tid; i < N; i += kQpThreads) {
    const double xu = q.Dz[i] * q.x[i];
    nx[i] = xu;
    q.v1[i] = xu;  // unscaled solution for the model-value pass
    p.ws_x[static_cast<size_t>(b) * N + i] = xu;
    p.ws_yb[static_cast<size_t>(b) * N + i] = q.cinv * (q.beta[i] / q.Dz[i]) * q.yb[i];
  }
  __syncthreads();
  for (int r = tid; r < nr; r += kQpThreads) {
    double* R = q.R(r);
    double* F = q.F(r);
    const int* I = q.I(r);
    const int aux = I[RI_AUX];
    F[R_Y] = q.cinv * F[R_E] * F[R_Y];
    for (int k = 0; k < 2; ++k) {
      F[R_XA0 + k] = (k < aux) ? F[R_DA0 + k] * F[R_XA0 + k] : 0.0;
      F[R_YA0 + k] = (k < aux) ? q.cinv * F[R_EA0 + k] * F[R_YA0 + k] : 0.0;
    }
    double val = F[R_C];
    for (int i = 0; i < I[RI_CNT]; ++i) val += R[i] * q.v1[I[RI_BASE] + i * I[RI_STRIDE]];
    // ConvexConstraints::violations (modeling.cpp:132-142) for constraint rows; hinge/abs cost = w * aux values
    F[R_MV] = (aux == AUX_ABS || aux == AUX_NONE) ? fabs(val) : fmax(val, 0.0);
  }
  __syncthreads();
  for (int oi = tid; oi < n_obj; oi += kQpThreads) {  // per object sums, canonical order, one thread per object
    const bool is_cnt = oi >= p.n_costs;
    double s = 0.0;
    if (!is_cnt && p.cost_objs[oi].kind == OBJ_JOINT_EQ_COST) s = joint_obj_value(p, p.cost_objs[oi], q.v1);  // exact quadratic
    for (int r = obj_start[oi]; r < obj_start[oi + 1]; ++r) {
      const double* F = q.F(r);
      if (is_cnt) s += F[R_MV];
      else s += F[R_W] * (F[R_XA0] + F[R_XA1]);  // ConvexObjective::value: the penalty terms use the aux values
    }
    if (is_cnt) p.model_cnt_viols[static_cast<size_t>(b) * p.n_cnts + (oi - p.n_costs)] = s;
    else p.model_cost_vals[static_cast<size_t>(b) * p.n_costs + oi] = s;
  }
  __syncthreads();
  if (rows_in_smem)  // the unscaled primal / dual row state is the next QP's warm start
    for (int t = tid; t < nr * q.RS; t += kQpThreads) rows_g[t] = rows_s[t];
  if (tid == 0) {
    // status map of osqp_interface.cpp:565-614
    int cvx = 2;
    if (res.status == QPS_SOLVED || res.status == QPS_SOLVED_INACC) cvx = 0;
    else if (res.status >= QPS_PINF && res.status <= QPS_DINF_INACC) cvx = 1;
    p.qp_status[b] = cvx;
    meta[0] = n_aux; meta[1] = nr; meta[2] = nnzA; meta[3] = (cvx == 0) ? 1 : 0; meta[4] = 0;
    p.ws_rho[b] = res.rho;
    if (!x_override) {
      p.n_admm_iters[b] += res.iters;
      p.qp_done[b] = 1;
    }
    if (admm_iters_out) admm_iters_out[b] = res.iters;
    if (polish_out) polish_out[b] = res.polish;
    if (p.qp_paths) {  // (off unless tb200_debug_enable_qp_paths)
      const QpPlan pl = qp_plan(DD <= 7, q.pinv, q.rows_smem, q.M, NB, p.qp_fast_passes != 0);
      int bits = qp_plan_block(pl, q.rows_smem) | (pl.fuse ? QPP_FUSED_CHECK : 0);
      if (res.pol_factor_ok == 1) bits |= pl.fast_polish ? QPP_POLISH_FAST : QPP_POLISH_GENERIC;
      if (FG || !S.factor_smem) bits |= QPP_FACTOR_GLOBAL;
      if (!S.pband_smem) bits |= QPP_BAND_GLOBAL;
      if (!rows_in_smem) bits |= QPP_ROWS_GLOBAL;
      atomicOr(&p.qp_paths[b], bits);
    }
    double* g = p.dbg + static_cast<size_t>(b) * 16;
    g[0] = res.status; g[1] = res.iters; g[2] = res.polish; g[3] = res.rho; g[4] = res.pri_res; g[5] = res.dua_res;
    g[6] = res.pol_pri; g[7] = res.pol_dua; g[8] = res.c; g[9] = res.pol_factor_ok; g[10] = res.rho_updates;
    g[11] = nr; g[12] = n_aux; g[13] = nnzA; g[14] = warm ? 1 : 0; g[15] = res.rounds;
  }
}

}  // namespace tb200
