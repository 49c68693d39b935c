// Batched convexify + exact evaluation + trust-region decision kernel (one CTA per trajectory).
//
// For every trajectory of the batch this kernel does, at one iterate, what the reference spreads over
//   costs[i]->convex(x) / cnts[i]->convex(x)                 trajopt_sco/src/optimizers.cpp:781-783
//   evaluateCosts / evaluateConstraintViols at new_x         optimizers.cpp:411-412 (merit evaluation)
//   the accept / shrink / converge / penalty decisions       optimizers.cpp:811-968
// in a single pass (the reference's 2-entry collision cache, collision_terms.hpp:216, exists only to
// share one FK + contact pass between value(new_x) and the next convex(new_x); here both are one pass).
// Outputs are the fixed-layout rows of DESIGN.md §3: CartPose error/Jacobian rows and the dense
// candidate collision rows {grad[D], dist0, margin, coeff|0}.
#pragma once
#include "joint_terms.cuh"
#include "kinematics.cuh"

namespace tb200 {

constexpr int kEvalThreads = 256;
enum EvalMode { EVAL_INIT = 0, EVAL_STEP = 1, EVAL_ONLY = 2 };

// Frames of the waypoint FK in shared memory: 13 doubles apart (12 used) and an odd number of doubles per waypoint, so
// that lanes working on different frames / waypoints hit different banks (12 and S*12 doubles are multiples of the
// bank period for the access patterns of the chain products: every lane landed on the same banks).
constexpr int kFrameStride = 13;
__host__ __device__ inline int eval_job_stride(int S) { return (S * kFrameStride) | 1; }

struct EvalSmem {
  // offsets in doubles into the dynamic shared buffer
  int x, sph, spo, jax, velp, objv, mask, misc, fr, terms, obst, sphr, segs, sphs, cobj, aobj, wscr, wscr_stride, cfk, sing, total;
};
// per-warp scratch of the AvoidSingularity objects: J(q) column by column ([D][6]), then u[6] and v[D] of its smallest
// singular value
__host__ __device__ inline int sing_scratch_stride(int D) { return (7 * D + 6 + 1) & ~1; }
// n_vel_objs: CartVel step pairs; cast: the collision objects are step pairs (continuous evaluator), each holding at
// most cast_cap active contacts; n_sing_objs: AvoidSingularity objects (their scratch is planned only when there are any)
__host__ __device__ inline EvalSmem eval_smem_layout(int T, int D, int L, int n_coll_objs, int n_mask_words, int S,
                                                      int n_joint_objs, int n_vel_objs, int cast, int cast_cap, int n_objs,
                                                      int n_sing_objs = 0) {
  EvalSmem s;
  int o = 0;
  s.x = o;      o += T * D;
  s.sph = o;    o += T * L * 3;                       // sphere centres per waypoint
  s.spo = o;    o += cast ? T * L * 3 : 0;            // centre - link origin (R_link * c_local) per waypoint
  o += o & 1;                                         // 16-byte alignment (vector loads)
  s.jax = o;    o += T * D * 6;                       // per (waypoint, joint): A[3], B[3] (see the kernel)
  s.obst = o;   o += 4 * 64;                          // this trajectory's obstacle spheres (x, y, z, r)
  s.sphr = o;   o += L + (L & 1);                     // radii of the robot spheres
  s.segs = o;   o += S * static_cast<int>(sizeof(DevSegment) / 8);   // the robot tables, read by every phase
  s.sphs = o;   o += L * static_cast<int>(sizeof(DevSphere) / 8);
  s.cobj = o;   o += n_coll_objs * static_cast<int>(sizeof(DevObj) / 8);   // the collision objects in kernel order
  s.aobj = o;   o += n_objs * static_cast<int>(sizeof(DevObj) / 8);        // every object: costs, then constraints
  s.velp = o;   o += n_vel_objs * 6;                  // link position at both waypoints of a CartVel pair
  s.objv = o;   o += n_coll_objs + n_joint_objs;      // exact value of every collision / joint-space object (in-order sums)
  s.mask = o;   o += n_mask_words;
  s.misc = o;   o += 8;
  o += o & 1;
  // per-warp scratch of the cast collision objects: one set of frames, the sphere centres at the two ends of the
  // running sub-segment, one joint vector (the contacts found so far live in a per-warp block of global memory:
  // EvalExtra::cast_scratch)
  (void)cast_cap;
  s.wscr_stride = cast ? (S * 12 + 2 * L * 3 + (L & 1) + ((D + 1) & ~1)) : 0;
  s.wscr = o;   o += 8 * s.wscr_stride;
  s.cfk = o;    o += 8 * (1 + D) * kFrameStride;    // running frames of the CartPose chain FK: one per lane and warp
  o += o & 1;
  s.terms = o;  o += n_joint_objs * 2 * T * D;        // per-(step, joint) terms of the joint-space objects
  o += o & 1;
  // the FK frames are dead once the joint axes / sphere centres are emitted: while the collision rows are written
  // their space holds the per-warp staging tiles of the row stores
  s.fr = o;                                           // frames of every FK job: local, then (in place) world
  const int a = T * eval_job_stride(S);
  const int st = (((D + 3) & 1) == 0 && !cast) ? 8 * 32 * (D + 3) : 0;  // one staging tile (32 rows) per warp
  o += a > st ? a : st;
  o += o & 1;
  s.sing = o;   o += n_sing_objs > 0 ? (kEvalThreads / 32) * sing_scratch_stride(D) : 0;
  s.total = o;
  return s;
}

struct EvalExtra {
  int n_cart_objs, n_coll_objs, n_joint_objs, n_vel_objs;
  int cast, cast_cap;                // cast: the collision objects are step pairs (continuous evaluator), each with room
                                     // for cast_cap active contacts (rows)
  double* cast_scratch;              // [gridDim * 8 warps][4 * cast_cap]: per contact (s, dist), key + rank, value in canonical order
  int* work_counter;                 // stand-alone launches: next trajectory to take (reset to 0 before every launch)
  const int* link_chain;             // [S][kMaxSeg + 1]: per segment, the number of segments on its chain from the root,
                                     // then the chain itself (root first, the segment last)
  const DevObj* vel_objs;            // CartVel step pairs
  int joint_seg[kMaxDof];            // segment that carries trajectory column j
  int joint_obj_idx[8];  // positions of the joint-space objects in the (costs, cnts) list
  const DevObj* cart_objs;   // list_index = index in its own list (cost / cnt), is_cnt says which list
  const DevObj* coll_objs;
  int qtype[kMaxDof];                // joint type per trajectory column
  unsigned sphere_jmask[kMaxSpheres];  // which columns move each sphere
  // SQP iteration log (tb200_problem_set_sqp_log; DESIGN.md section 4.7), nullptr: off.  One record per QP solve plus the
  // state after the initial evaluation, [B][log_cap][log_stride] doubles; records past log_cap are counted, not written.
  // (Here rather than in DevProblem: a larger DevProblem changes the register allocation of the QP step.)
  double* log;
  int* log_len;                // [B] records written
  int* log_dropped;            // [B] records that did not fit
  int log_cap, log_stride, log_with_x, pad;
  // AvoidSingularity objects (one per step; coeff: the term's coefficient, margin: its lambda)
  const DevObj* sing_objs;
  int n_sing_objs, pad_sing;
  // Optimizer parameters, [B]: trajectory b runs under sqp[b] (tb200_problem_set_sqp_params / _per_traj fill every row).
  // sqp_timed: some row has a time limit (max_time < DBL_MAX); the clock check at the iteration top is one uniform branch.
  const SqpParams* sqp;
  int sqp_timed, pad_sqp;
};

#ifdef TB200_EVAL_PROFILE
// cycles of thread 0 between the block barriers of eval_step, summed over CTAs (scripts/eval_phases.py)
static __device__ unsigned long long g_eval_prof[16];
static __device__ unsigned long long g_eval_trace[3 * 4096];  // per CTA: start ns, end ns, SM id
#define EVAL_PROF(k) do { if (threadIdx.x == 0) { const long long now_ = clock64(); atomicAdd(&g_eval_prof[k], (unsigned long long)(now_ - prof_t_)); prof_t_ = now_; } } while (0)
#define EVAL_PROF_BEGIN()                                                                          \
  long long prof_t_ = clock64();                                                                   \
  if (threadIdx.x == 0 && b < 4096) {                                                              \
    unsigned long long t_;                                                                         \
    unsigned sm_;                                                                                  \
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_));                                         \
    asm volatile("mov.u32 %0, %smid;" : "=r"(sm_));                                               \
    g_eval_trace[3 * b] = t_;                                                                      \
    g_eval_trace[3 * b + 2] = sm_;                                                                 \
  }
#define EVAL_PROF_END()                                                                            \
  if (threadIdx.x == 0 && b < 4096) {                                                              \
    unsigned long long t_;                                                                         \
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_));                                         \
    g_eval_trace[3 * b + 1] = t_;                                                                  \
  }
#else
#define EVAL_PROF_END()
#define EVAL_PROF(k)
#define EVAL_PROF_BEGIN()
#endif

// FK of ONE joint state by a warp: local frames (lanes over segments), then the chain products row by row
// (lanes 0-2; the other lanes only keep the barriers).  F: [S][12] world frames (R row-major, p).
__device__ inline void warp_fk(const DevProblem& p, const double* q, double* F, int lane) {
  const int Sg = p.S;
  for (int sg = lane; sg < Sg; sg += 32) {
    const DevSegment g = p.segs[sg];
    Frame loc;
    segment_local_q(g, g.q_index >= 0 ? q[g.q_index] : 0.0, loc);
    double* f = F + sg * 12;
    for (int i = 0; i < 9; ++i) f[i] = loc.R[i];
    for (int i = 0; i < 3; ++i) f[9 + i] = loc.p[i];
  }
  __syncwarp();
  const bool act = lane < 3;
  const int i = act ? lane : 0;
  for (int sg = 0; sg < Sg; ++sg) {
    const int parent = p.segs[sg].parent;
    double l[12];
    for (int k = 0; k < 12; ++k) l[k] = F[sg * 12 + k];
    __syncwarp();  // every row has read the local frame before it is overwritten
    if (act && parent >= 0) {
      const double* P = F + parent * 12;
      const double r0 = P[i * 3], r1 = P[i * 3 + 1], r2 = P[i * 3 + 2], pi = P[9 + i];
      F[sg * 12 + i * 3 + 0] = r0 * l[0] + r1 * l[3] + r2 * l[6];
      F[sg * 12 + i * 3 + 1] = r0 * l[1] + r1 * l[4] + r2 * l[7];
      F[sg * 12 + i * 3 + 2] = r0 * l[2] + r1 * l[5] + r2 * l[8];
      F[sg * 12 + 9 + i] = r0 * l[9] + r1 * l[10] + r2 * l[11] + pi;
    }
    __syncwarp();
  }
}

// 8-byte asynchronous copy global -> shared (LDGSTS): the copies of one phase are all in flight together instead of
// each loop's store waiting for its own load
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// The SQP log record of a decision without its outcome (eval_step_impl; DESIGN.md section 4.7).  A function of its own so
// that the decision code is compiled as without the log.
static __device__ __noinline__ void log_record_arrays(const DevProblem& p, const EvalExtra& ex, const int mode, const int b,
                                               const bool qp_failed, const DevObj* aobjs, const double* out_cost,
                                               const double* out_viol, const double* xs) {
  const int tid = threadIdx.x;
  const int n = ex.log_len[b];
  if (!(mode == EVAL_INIT || !(ex.cast && p.lvs_overflow[b])) || n >= ex.log_cap) return;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  const int nc = p.n_costs, nk = p.n_cnts;
  double* rec = ex.log + (static_cast<size_t>(b) * ex.log_cap + n) * ex.log_stride;
  if (tid == 0) {
    const bool qp = mode == EVAL_STEP;
    const double* g = p.dbg + static_cast<size_t>(b) * 16;
    rec[LOG_KIND] = qp ? 1 : 0;
    rec[LOG_ROUND] = p.merit_round[b]; rec[LOG_ITER] = p.sqp_iter[b]; rec[LOG_TRUST] = p.trust[b];
    rec[LOG_OLD_MERIT] = rec[LOG_MODEL_MERIT] = rec[LOG_NEW_MERIT] = qnan;
    rec[LOG_QP_STATUS] = qp ? g[0] : qnan; rec[LOG_ADMM_ITERS] = qp ? g[1] : qnan; rec[LOG_ACTION] = -1;
    rec[LOG_PRI_RES] = qp ? g[4] : qnan; rec[LOG_DUA_RES] = qp ? g[5] : qnan; rec[LOG_RHO] = qp ? g[3] : qnan;
    rec[LOG_POLISH] = qp ? g[2] : qnan; rec[LOG_WARM] = qp ? g[14] : qnan;
  }
  rec += kLogHeader;
  const double* mu = p.merit_coeffs + static_cast<size_t>(b) * nk;
  const double* mc = p.model_cost_vals + static_cast<size_t>(b) * nc;
  const double* mk = p.model_cnt_viols + static_cast<size_t>(b) * nk;
  const bool model = mode == EVAL_STEP && !qp_failed;
  for (int i = tid; i < nk; i += kEvalThreads) rec[i] = mu[i];
  rec += nk;
  for (int i = tid; i < nc; i += kEvalThreads)  // as summed into model_merit: quadratic joint costs are exact
    rec[i] = model ? (aobjs[i].kind == OBJ_JOINT_EQ_COST ? out_cost[i] : mc[i]) : qnan;
  rec += nc;
  for (int i = tid; i < nk; i += kEvalThreads) rec[i] = model ? mk[i] : qnan;
  rec += nk;
  for (int i = tid; i < nc; i += kEvalThreads) rec[i] = qp_failed ? qnan : out_cost[i];
  rec += nc;
  for (int i = tid; i < nk; i += kEvalThreads) rec[i] = qp_failed ? qnan : out_viol[i];
  rec += nk;
  if (ex.log_with_x)
    for (int i = tid; i < p.N; i += kEvalThreads) rec[i] = qp_failed ? qnan : xs[i];
}

// ---- AvoidSingularity rows (kinematic_terms.cpp:586-642) ------------------------------------------------------------
// err = 1/(s + lambda) - 1/(0.1 + lambda) with s the smallest singular value of the 6 x D geometric Jacobian J(q) of the
// link's origin (linear rows, then angular; a zero column for a joint that does not move the link), and the gradient
// g_j = u' ((J(q + eps e_j) - J(q)) / eps) v * (-1 / (s + lambda)^2), eps = 1e-6, with u, v the singular vectors of s.
// Both go out scaled by the term's coefficient: one row of the Cartesian buffers per object.
constexpr double kSingEps = 1e-6;      // AvoidSingularityJacCalculator's eps_
// Jacobi rotations stop when every |a_p . a_q| <= M eps |a_p| |a_q| (M: the length of the columns; LAPACK's dgesvj
// uses the same scale): below that the off-diagonal is the rounding of the dot product itself
constexpr double kSingSvdEps = 2.220446049250313e-16;
constexpr int kSingSvdSweeps = 32;

// the chain of a link at q + eps e_pj (pj < 0: at q), running frame in registers with the products of the CartPose
// walk; on_joint(segment, R, p) sees the world frame of every joint segment on the chain.  Returns the link origin.
template <class OnJoint>
__device__ __forceinline__ void sing_walk(const DevSegment* segs, const int* chain, const double* qw, const int pj,
                                          double* pe, OnJoint&& on_joint) {
  double R[9], P[3];
  const int clen = chain[0];
  for (int k = 0; k < clen; ++k) {
    const DevSegment& g = segs[chain[1 + k]];
    const double qv = (g.q_index >= 0) ? qw[g.q_index] + (g.q_index == pj ? kSingEps : 0.0) : 0.0;
    Frame loc;
    segment_local_q(g, qv, loc);
    if (k == 0) {
#pragma unroll
      for (int i = 0; i < 9; ++i) R[i] = loc.R[i];
#pragma unroll
      for (int i = 0; i < 3; ++i) P[i] = loc.p[i];
    } else {
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double r0 = R[i * 3], r1 = R[i * 3 + 1], r2 = R[i * 3 + 2], rp = P[i];
        R[i * 3 + 0] = r0 * loc.R[0] + r1 * loc.R[3] + r2 * loc.R[6];
        R[i * 3 + 1] = r0 * loc.R[1] + r1 * loc.R[4] + r2 * loc.R[7];
        R[i * 3 + 2] = r0 * loc.R[2] + r1 * loc.R[5] + r2 * loc.R[8];
        P[i] = r0 * loc.p[0] + r1 * loc.p[1] + r2 * loc.p[2] + rp;
      }
    }
    if (g.q_index >= 0) on_joint(g, R, P);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) pe[i] = P[i];
}

// column of the geometric Jacobian at the link origin pe for a joint with world frame (R, P): [a x (pe - o); a]
// (revolute) or [a; 0] (prismatic), a = R * axis, o = P
__device__ __forceinline__ void sing_column(const DevSegment& g, const double* R, const double* P, const double* pe,
                                            double* col) {
  double a[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) a[i] = R[i * 3] * g.axis[0] + R[i * 3 + 1] * g.axis[1] + R[i * 3 + 2] * g.axis[2];
  if (g.joint_type == 1) {
    const double d0 = pe[0] - P[0], d1 = pe[1] - P[1], d2 = pe[2] - P[2];
    col[0] = a[1] * d2 - a[2] * d1; col[1] = a[2] * d0 - a[0] * d2; col[2] = a[0] * d1 - a[1] * d0;
    col[3] = a[0]; col[4] = a[1]; col[5] = a[2];
  } else {
    col[0] = a[0]; col[1] = a[1]; col[2] = a[2];
    col[3] = 0.0; col[4] = 0.0; col[5] = 0.0;
  }
}

// sum over the warp, the same bits in every lane (lane 0's butterfly result, broadcast)
__device__ __forceinline__ double sing_warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return __shfl_sync(0xffffffffu, v, 0);
}

// One warp per object (objects warp, warp + 8, ...).  Lane 0 builds J(q) in shared memory; the warp runs a one-sided
// Jacobi SVD on it (on J's D columns when D < 6, else on the 6 columns of J', one row of the rotated matrix per lane,
// rotations in a fixed cyclic order); lane 1 + j then walks the chain at q + eps e_j and projects its difference
// columns on u, v as it meets them.  Called only by the SING instances of the evaluation step.
template <int DD>
static __device__ __noinline__ void singularity_objects(const EvalExtra& ex, const double* xs, const DevSegment* segs,
                                                        double* scratch, double* err_out, double* jac_out, const int stride) {
  constexpr int D = DD;
  constexpr int NC = D < 6 ? D : 6;  // columns the rotations act on
  constexpr int M = D < 6 ? 6 : D;   // their length
  constexpr double tol = M * kSingSvdEps;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* J0 = scratch + warp * sing_scratch_stride(D);
  double* uu = J0 + 6 * D;
  double* vv = uu + 6;
  for (int c = warp; c < ex.n_sing_objs; c += kEvalThreads / 32) {
    const DevObj& o = ex.sing_objs[c];
    const int* chain = ex.link_chain + o.link * (kMaxSeg + 1);
    const double* qw = xs + o.first * D;
    const int pj = lane - 1;  // lane 0: J(q); lane 1 + j: J(q + eps e_j)
    const bool work = lane <= D;
    double pe[3] = {0.0, 0.0, 0.0};
    if (work) sing_walk(segs, chain, qw, pj, pe, [](const DevSegment&, const double*, const double*) {});
    for (int i = lane; i < 6 * D; i += 32) J0[i] = 0.0;
    __syncwarp();
    if (lane == 0)
      sing_walk(segs, chain, qw, -1, pe, [&](const DevSegment& g, const double* R, const double* P) {
        sing_column(g, R, P, pe, J0 + 6 * g.q_index);
      });
    __syncwarp();
    // ---- one-sided Jacobi: A V = W with orthogonal columns; A = J (D < 6) or J' (D >= 6), lane i holds row i ----
    double a[NC], vr[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      a[k] = lane < M ? (D < 6 ? J0[k * 6 + lane] : J0[lane * 6 + k]) : 0.0;
      vr[k] = (lane == k) ? 1.0 : 0.0;
    }
    for (int sweep = 0; sweep < kSingSvdSweeps; ++sweep) {
      bool rotated = false;
#pragma unroll
      for (int pa = 0; pa < NC - 1; ++pa) {
#pragma unroll
        for (int qa = pa + 1; qa < NC; ++qa) {
          const double al = sing_warp_sum(a[pa] * a[pa]), be = sing_warp_sum(a[qa] * a[qa]), ga = sing_warp_sum(a[pa] * a[qa]);
          if (fabs(ga) > tol * sqrt(al * be)) {  // (warp-uniform)
            const double zeta = (be - al) / (2.0 * ga);
            const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
            const double ap = a[pa], aq = a[qa], vp = vr[pa], vq = vr[qa];
            a[pa] = cs * ap - sn * aq; a[qa] = sn * ap + cs * aq;
            vr[pa] = cs * vp - sn * vq; vr[qa] = sn * vp + cs * vq;
            rotated = true;
          }
        }
      }
      if (!rotated) break;
    }
    // the smallest singular value: the shortest column of W
    double sigma = 0.0, ak = 0.0, vk = 0.0;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
      const double sk = sqrt(sing_warp_sum(a[k] * a[k]));
      if (k == 0 || sk < sigma) { sigma = sk; ak = a[k]; vk = vr[k]; }
    }
    // s = 0 leaves the direction W_k / s undefined: that vector is taken as 0 (the gradient is then 0)
    const double wk = sigma > 0.0 ? ak / sigma : 0.0;
    if (D < 6) {  // u = W_k / s, v = V_k
      if (lane < 6) uu[lane] = wk;
      if (lane < D) vv[lane] = vk;
    } else {      // J' = W V': u = V_k, v = W_k / s
      if (lane < 6) uu[lane] = vk;
      if (lane < D) vv[lane] = wk;
    }
    __syncwarp();
    const double coeff = o.coeff, lam = o.margin;
    if (lane == 0) err_out[o.src_off] = coeff * (1.0 / (sigma + lam) - 1.0 / (0.1 + lam));
    if (work && lane > 0) {
      double g = 0.0, pk[3];  // (pe: this lane's link origin from the first walk)
      sing_walk(segs, chain, qw, pj, pk, [&](const DevSegment& sg, const double* R, const double* P) {
        double col[6];
        sing_column(sg, R, P, pe, col);
        const double* c0 = J0 + 6 * sg.q_index;
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i) s += uu[i] * ((col[i] - c0[i]) / kSingEps);
        g += s * vv[sg.q_index];
      });
      g *= -1.0 / ((sigma + lam) * (sigma + lam));
      jac_out[static_cast<size_t>(o.src_off) * stride + pj] = coeff * g;
    }
    __syncwarp();  // the scratch of the warp is reused by its next object
  }
}

// SING: the instance for problems with AvoidSingularity objects (every other problem runs SING = 0, whose code has
// none of the term's)
template <int DD, int SING>
__device__ __forceinline__ void eval_step_impl(const DevProblem& p, const EvalExtra& ex, const int mode, const int b,
                                               const double* x_in /*EVAL_ONLY*/, bool& tables_ready) {
  extern __shared__ double sm[];
  const int tid = threadIdx.x;
  constexpr int D = DD;
  EVAL_PROF_BEGIN();
  const int T = p.T, N = p.N, L = p.L, O = p.O;
  if (mode != EVAL_ONLY && p.status[b] != 5 /*running == INVALID*/) return;
  if (mode == EVAL_STEP && p.qp_done[b] == 0) return;  // (defensive: the QP step of this trajectory has not finished)
  const bool qp_failed = (mode == EVAL_STEP) && (p.qp_status[b] != 0);
  if (tid == 0 && !qp_failed) atomicAdd(p.active_count + 1, 1);  // trajectories actually convexified (bench: bytes moved)
  const int n_mask_words = p.n_coll_objs * p.coll_words;
  const EvalSmem S = eval_smem_layout(T, D, L, p.n_coll_objs, n_mask_words, p.S, ex.n_joint_objs, ex.n_vel_objs,
                                      ex.cast, ex.cast_cap, p.n_costs + p.n_cnts, SING ? ex.n_sing_objs : 0);
  static_assert(sizeof(DevObj) % 8 == 0 && sizeof(DevSegment) % 8 == 0 && sizeof(DevSphere) % 8 == 0, "tables are copied as doubles");
  const DevObj* cobjs = reinterpret_cast<const DevObj*>(sm + S.cobj);
  const DevObj* aobjs = reinterpret_cast<const DevObj*>(sm + S.aobj);
  double* xs = sm + S.x;
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(sm + S.mask);
  int* misc = reinterpret_cast<int*>(sm + S.misc);

  // destination convexification buffer: the one NOT holding the rows of the current iterate
  const int cur = (mode == EVAL_ONLY) ? 1 : p.cur_buf[b];
  const int dst = (mode == EVAL_STEP) ? 1 - cur : ((mode == EVAL_INIT) ? 0 : 0);
  const size_t slot = static_cast<size_t>(dst) * p.B + b;

  if (!qp_failed) {
    // ---- load the iterate (coalesced) -------------------------------------------------------
    const double* src = (mode == EVAL_ONLY) ? x_in + static_cast<size_t>(b) * N
                                            : (mode == EVAL_INIT ? p.init_traj : p.new_x) + static_cast<size_t>(b) * N;
    for (int i = tid; i < N; i += kEvalThreads) cp_async8(xs + i, src + i);
    for (int i = tid; i < n_mask_words; i += kEvalThreads) mask[i] = 0ull;
    if (tid == 0) {
      misc[2] = 0;  // work counter of the row phase
      misc[3] = 0;  // ... of the CartPose objects
    }
    {
      const double* og = p.obstacles + (p.obstacles_per_traj ? static_cast<size_t>(b) * O * 4 : 0);
      for (int i = tid; i < O * 4; i += kEvalThreads) cp_async8(sm + S.obst + i, og + i);
    }
    if (!tables_ready) {  // the same for every trajectory: a persistent CTA of the stand-alone kernel copies them once
      tables_ready = true;
      for (int i = tid; i < L; i += kEvalThreads) cp_async8(sm + S.sphr + i, &p.spheres[i].r);
      const double* sg_g = reinterpret_cast<const double*>(p.segs);
      for (int i = tid; i < p.S * static_cast<int>(sizeof(DevSegment) / 8); i += kEvalThreads) cp_async8(sm + S.segs + i, sg_g + i);
      const double* sp_g = reinterpret_cast<const double*>(p.spheres);
      for (int i = tid; i < L * static_cast<int>(sizeof(DevSphere) / 8); i += kEvalThreads) cp_async8(sm + S.sphs + i, sp_g + i);
      constexpr int OD = static_cast<int>(sizeof(DevObj) / 8);
      const double* co_g = reinterpret_cast<const double*>(ex.coll_objs);
      for (int i = tid; i < p.n_coll_objs * OD; i += kEvalThreads) cp_async8(sm + S.cobj + i, co_g + i);
      const double* cs_g = reinterpret_cast<const double*>(p.cost_objs);
      for (int i = tid; i < p.n_costs * OD; i += kEvalThreads) cp_async8(sm + S.aobj + i, cs_g + i);
      const double* cn_g = reinterpret_cast<const double*>(p.cnt_objs);
      for (int i = tid; i < p.n_cnts * OD; i += kEvalThreads) cp_async8(sm + S.aobj + p.n_costs * OD + i, cn_g + i);
    }
    cp_async_wait_all();
    if (mode == EVAL_INIT)  // getClosestFeasiblePoint quirk, modeling.cpp:267-268 (a thread clamps what it copied itself)
      for (int i = tid; i < N; i += kEvalThreads) xs[i] = fmin(p.upper[i % D] - 1e-3, xs[i]);
    __syncthreads();
    EVAL_PROF(1);

    // ---- FK: one job per waypoint (the perturbed states of the CartPose objects are handled by their own warps) ---
    // (1) local frames of every (job, segment) in parallel (this is where the sincos are), (2) the chain
    // products, one lane per (job, frame row): row i of a world frame depends only on row i of the parent's,
    // so the three lanes of a job never wait for each other, (3) emission of what the row writers need.
    // Head start: the CartPose objects need the iterate only, and one of them is a long dependent chain (chain FK of eight
    // states, pose error, atan2) that used to set the length of the row phase.  So when the problem has any, warp 7 starts
    // on them right away while warps 0-6 run the three FK phases among themselves (named barrier 1, 224 threads); warp 7
    // waits for the end of the emission (barrier 2: 224 arrive, 32 wait) before it touches anything the FK produced.
    const bool head = ex.n_cart_objs > 0;
    const int nthr = head ? kEvalThreads - 32 : kEvalThreads;
    const bool fk_thread = tid < nthr;
    auto fk_sync = [&]() {
      if (head) asm volatile("bar.sync 1, 224;" ::: "memory");
      else __syncthreads();
    };
    const int n_jobs = T, Sg = p.S;
    double* FR = sm + S.fr;
    constexpr int FS = kFrameStride;
    const int JS = eval_job_stride(Sg);
    const DevSegment* segs = reinterpret_cast<const DevSegment*>(sm + S.segs);
    const DevSphere* sphs = reinterpret_cast<const DevSphere*>(sm + S.sphs);
    double* const terms = sm + S.terms;
    if (fk_thread) {
    for (int w = tid; w < n_jobs * Sg; w += nthr) {
      const int job = w / Sg, sg = w % Sg;
      const DevSegment& g = segs[sg];
      const double qv = (g.q_index >= 0) ? xs[job * D + g.q_index] : 0.0;
      Frame loc;
      segment_local_q(g, qv, loc);
      double* f = FR + job * JS + sg * FS;
      for (int i = 0; i < 9; ++i) f[i] = loc.R[i];
      for (int i = 0; i < 3; ++i) f[9 + i] = loc.p[i];
    }
    // joint-space terms (they need the iterate only): slot j of the term buffer belongs to the j-th joint-space object in
    // (costs, cnts) order; their in-order sums are work items of the row phase below
    for (int slot_j = 0; slot_j < ex.n_joint_objs; ++slot_j) {
      const int i = ex.joint_obj_idx[slot_j];
      const DevObj& o = aobjs[i];
      const DevJointTerm& jt = p.joint_terms[o.term];
      double* tb = terms + static_cast<size_t>(slot_j) * 2 * T * D;
      const int kind = o.kind, order = o.order, first = o.first;
      for (int w = tid; w < o.n_steps * D; w += nthr) {
        const int t = first + w / D, d = w % D;
        const double e = joint_err(xs, D, order, t, d, jt.targets[d]);
        double v0, v1 = 0.0;
        if (kind == OBJ_JOINT_EQ_COST) v0 = e * e * jt.coeffs[d];
        else if (kind == OBJ_JOINT_EQ_CNT) v0 = fabs(e * e * jt.coeffs[d]);  // value() is c*e^2 while the row is c*e (trajectory_costs.cpp:160 vs 173)
        else {
          v0 = fmax((e - jt.upper[d]) * jt.coeffs[d], 0.0);
          v1 = fmax((jt.lower[d] - e) * jt.coeffs[d], 0.0);
        }
        tb[2 * w] = v0;
        tb[2 * w + 1] = v1;
      }
    }
    }
    if (fk_thread) fk_sync();
    EVAL_PROF(2);
    if (fk_thread) {
    for (int w = tid; w < ((n_jobs * 4 + 31) & ~31); w += nthr) {  // whole warps: __syncwarp below
      // four lanes per job (three rows + one idle) so that the rows of a job always sit in the same warp.  A lane
      // only ever needs ITS row of the parent frame: along a chain (parent == previous segment) it is still in
      // registers, at a branch point it reads back what it wrote itself.  The one barrier per step keeps the
      // in-place overwrite of a local frame behind its readers.
      const bool act = w < n_jobs * 4 && (w & 3) < 3;
      const int job = (w < n_jobs * 4) ? w / 4 : 0, i = (w & 3) % 3;
      double* F = FR + job * JS;
      double r0 = 0.0, r1 = 0.0, r2 = 0.0, rp = 0.0;
      for (int sg = 0; sg < Sg; ++sg) {
        const int parent = segs[sg].parent;
        double l[12];
        for (int k = 0; k < 12; ++k) l[k] = F[sg * FS + k];
        __syncwarp();
        if (parent >= 0) {
          if (parent != sg - 1) {
            const double* P = F + parent * FS;
            r0 = P[i * 3]; r1 = P[i * 3 + 1]; r2 = P[i * 3 + 2]; rp = P[9 + i];
          }
          const double n0 = r0 * l[0] + r1 * l[3] + r2 * l[6], n1 = r0 * l[1] + r1 * l[4] + r2 * l[7],
                       n2 = r0 * l[2] + r1 * l[5] + r2 * l[8], np = r0 * l[9] + r1 * l[10] + r2 * l[11] + rp;
          r0 = n0; r1 = n1; r2 = n2; rp = np;
          if (act) {
            F[sg * FS + i * 3 + 0] = r0;
            F[sg * FS + i * 3 + 1] = r1;
            F[sg * FS + i * 3 + 2] = r2;
            F[sg * FS + 9 + i] = rp;
          }
        } else {  // a root segment: its world frame is its local frame
          r0 = (i == 0) ? l[0] : ((i == 1) ? l[3] : l[6]);  // (selects, not l[3 * i]: the frame stays in registers)
          r1 = (i == 0) ? l[1] : ((i == 1) ? l[4] : l[7]);
          r2 = (i == 0) ? l[2] : ((i == 1) ? l[5] : l[8]);
          rp = (i == 0) ? l[9] : ((i == 1) ? l[10] : l[11]);
        }
      }
    }
    }
    if (fk_thread) fk_sync();
    EVAL_PROF(3);
    if (fk_thread) {
    // per (waypoint, joint) the two vectors the gradient of a point on the chain needs: for a point c and a unit
    // direction n,  n . d(c)/dq_j = n . (a_j x (c - o_j)) = A_j . (c x n) - B_j . n  with A_j = a_j, B_j = a_j x o_j
    // (revolute; a_j axis, o_j origin of the joint in the scene root) and A_j = 0, B_j = -a_j (prismatic).
    // Six doubles per (waypoint, joint), 16-byte aligned: the row writers read them as broadcasts.
    for (int w = tid; w < T * Sg; w += nthr) {
      const int t = w / Sg, sg = w % Sg;
      const DevSegment& g = segs[sg];
      if (g.q_index < 0) continue;
      const double* f = FR + t * JS + sg * FS;
      double* ab = sm + S.jax + (t * D + g.q_index) * 6;
      double a[3];
      for (int i = 0; i < 3; ++i) a[i] = f[i * 3] * g.axis[0] + f[i * 3 + 1] * g.axis[1] + f[i * 3 + 2] * g.axis[2];
      if (g.joint_type == 1) {
        const double ox = f[9], oy = f[10], oz = f[11];
        ab[0] = a[0]; ab[1] = a[1]; ab[2] = a[2];
        ab[3] = a[1] * oz - a[2] * oy; ab[4] = a[2] * ox - a[0] * oz; ab[5] = a[0] * oy - a[1] * ox;
      } else {
        ab[0] = 0.0; ab[1] = 0.0; ab[2] = 0.0;
        ab[3] = -a[0]; ab[4] = -a[1]; ab[5] = -a[2];
      }
    }
    for (int w = tid; w < T * L; w += nthr) {
      const int t = w / L, sl = w % L;
      const DevSphere& sp = sphs[sl];
      const double* f = FR + t * JS + sp.segment * FS;
      double* sph = sm + S.sph + w * 3;
      for (int i = 0; i < 3; ++i) {
        const double off = f[i * 3] * sp.c[0] + f[i * 3 + 1] * sp.c[1] + f[i * 3 + 2] * sp.c[2];
        sph[i] = off + f[9 + i];
        if (ex.cast) sm[S.spo + w * 3 + i] = off;
      }
    }
    for (int w = tid; w < ex.n_vel_objs * 6; w += nthr) {  // link position at both ends of a CartVel pair
      const int c = w / 6, k = (w % 6) / 3, i = w % 3;
      const DevObj& o = ex.vel_objs[c];
      sm[S.velp + w] = FR[(o.first + k) * JS + o.link * FS + 9 + i];
    }
    }
    if (fk_thread) {
      fk_sync();
      if (head) asm volatile("bar.arrive 2, 256;" ::: "memory");
    }
    EVAL_PROF(4);

    // ---- CartPose rows: error + forward-difference Jacobian (kinematic_terms.cpp:250-263, 348-366) ----
    // One warp per CartPose object, lane 0 the unperturbed state, lane 1+i the state q + eps e_i (DEFAULT_EPSILON,
    // kinematic_terms.hpp:14).  Every lane runs the FK of ITS state along the link's chain in registers (same products
    // in the same order as the waypoint FK above) and then the pose-error pipeline ONCE (a long dependent chain of fp64
    // divisions, square roots and an atan2); the base error reaches the difference quotients by shuffle.  No shared
    // memory per object, so a problem may carry any number of them (configs[4]: two per waypoint).
    auto cart_object = [&](const int c) {
      const int col = tid & 31;  // col 0 = error, col 1+i = Jacobian column i
      const bool work = col < 1 + D;
      const DevObj& o = ex.cart_objs[c];
      const DevCartTerm& ct = p.cart_terms[o.term];
      Frame tgt, off, lf, src, e1;
      {
        // the running frame lives in shared memory (one 13-double slot per lane), the segment's local frame in
        // registers: row i of (frame * local) needs only row i of the frame, so the product is formed in place
        const int* chain = ex.link_chain + o.link * (kMaxSeg + 1);
        const int clen = chain[0], pj = work ? col - 1 : -1;
        const double* qw = xs + o.first * D;
        double* cur = sm + S.cfk + ((tid >> 5) * (1 + D) + (work ? col : 0)) * kFrameStride;
        for (int k = 0; k < clen; ++k) {
          const DevSegment& g = segs[chain[1 + k]];
          const double qv = (g.q_index >= 0) ? qw[g.q_index] + (g.q_index == pj ? 1e-5 : 0.0) : 0.0;
          Frame loc;
          segment_local_q(g, qv, loc);
          if (work) {
            if (k == 0) {
#pragma unroll
              for (int i = 0; i < 9; ++i) cur[i] = loc.R[i];
#pragma unroll
              for (int i = 0; i < 3; ++i) cur[9 + i] = loc.p[i];
            } else {
#pragma unroll
              for (int i = 0; i < 3; ++i) {
                const double r0 = cur[i * 3], r1 = cur[i * 3 + 1], r2 = cur[i * 3 + 2], rp = cur[9 + i];
                cur[i * 3 + 0] = r0 * loc.R[0] + r1 * loc.R[3] + r2 * loc.R[6];
                cur[i * 3 + 1] = r0 * loc.R[1] + r1 * loc.R[4] + r2 * loc.R[7];
                cur[i * 3 + 2] = r0 * loc.R[2] + r1 * loc.R[5] + r2 * loc.R[8];
                cur[9 + i] = r0 * loc.p[0] + r1 * loc.p[1] + r2 * loc.p[2] + rp;
              }
            }
          }
        }
#pragma unroll
        for (int i = 0; i < 9; ++i) lf.R[i] = cur[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) lf.p[i] = cur[9 + i];
      }
      quat_to_frame(o.target_slot >= 0 ? p.cart_targets + (static_cast<size_t>(b) * p.n_cart_targets + o.target_slot) * 7 : ct.tgt, tgt);
      for (int i = 0; i < 9; ++i) off.R[i] = ct.src_R[i];
      for (int i = 0; i < 3; ++i) off.p[i] = ct.src_p[i];
      frame_mul(lf, off, src);
      rel_pose(tgt, src, e1);
      double a1[3], g1;
      rot_err_decomposed(e1.R, a1, g1);
      double a0[3], e0p[3];
      const double g0 = __shfl_sync(0xffffffffu, g1, 0);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        a0[i] = __shfl_sync(0xffffffffu, a1[i], 0);
        e0p[i] = __shfl_sync(0xffffffffu, e1.p[i], 0);
      }
      double* err_out = p.cart_err + slot * p.n_cart_rows + o.src_off;
      double* jac_out = p.cart_jac + (slot * p.n_cart_rows + o.src_off) * p.cart_stride;
      if (col == 0) {
        const double e0 = e1.p[0], e1v = e1.p[1], e2 = e1.p[2], e3 = a1[0] * g1, e4 = a1[1] * g1, e5 = a1[2] * g1;
        for (int r = 0; r < ct.n_idx; ++r) {  // (a select chain: a dynamically indexed array would live in local memory)
          const int ix = ct.idx[r];
          const double ev = ix == 0 ? e0 : (ix == 1 ? e1v : (ix == 2 ? e2 : (ix == 3 ? e3 : (ix == 4 ? e4 : e5))));
          err_out[r] = ev * ct.coeff[r];
        }
      } else if (work) {
        if (a1[0] * a0[0] + a1[1] * a0[1] + a1[2] * a0[2] < 0) {
          a1[0] = -a1[0]; a1[1] = -a1[1]; a1[2] = -a1[2];
          g1 = -g1;
        }
        const double diff = g1 - g0, pi = 3.14159265358979323846;
        if (diff > pi) g1 -= 2.0 * pi;
        else if (diff < -pi) g1 += 2.0 * pi;
        const double d0 = e1.p[0] - e0p[0], d1 = e1.p[1] - e0p[1], d2 = e1.p[2] - e0p[2], d3 = a1[0] * g1 - a0[0] * g0,
                     d4 = a1[1] * g1 - a0[1] * g0, d5 = a1[2] * g1 - a0[2] * g0;
        for (int r = 0; r < ct.n_idx; ++r) {
          const int ix = ct.idx[r];
          const double dv = ix == 0 ? d0 : (ix == 1 ? d1 : (ix == 2 ? d2 : (ix == 3 ? d3 : (ix == 4 ? d4 : d5))));
          jac_out[r * p.cart_stride + (col - 1)] = dv / 1e-5 * ct.coeff[r];
        }
      }
    };
    // the objects are handed out one at a time (a counter in shared memory): warp 7 takes them from the start, the others
    // join once the FK is done
    auto cart_objects = [&]() {
      for (;;) {
        int c = 0;
        if ((tid & 31) == 0) c = atomicAdd(&misc[3], 1);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c >= ex.n_cart_objs) break;
        cart_object(c);
      }
    };
    // (one copy of the code: warp 7 runs the loop twice — before and after it has waited for the emission of warps 0-6)
    for (int pass = (head && !fk_thread) ? 0 : 1; pass < 2; ++pass) {
      cart_objects();
      if (pass == 0) asm volatile("bar.sync 2, 256;" ::: "memory");
    }

    // ---- CartVel rows (kinematic_terms.cpp:376-425): err = [p1 - p0 - lim; p0 - p1 - lim], rows over (q_t, q_t+1)
    // with the translational geometric Jacobians J_k(:, j) = a_j x (p_k - o_j) = A_j x p_k - B_j ------------------
    for (int w = tid; w < ex.n_vel_objs * (2 * D + 6); w += kEvalThreads) {
      const int c = w / (2 * D + 6), e = w % (2 * D + 6);
      const DevObj& o = ex.vel_objs[c];
      const double* p0 = sm + S.velp + c * 6;
      const double* p1 = p0 + 3;
      double* err_out = p.cart_err + slot * p.n_cart_rows + o.src_off;
      double* jac_out = p.cart_jac + (slot * p.n_cart_rows + o.src_off) * p.cart_stride;
      if (e < 6) {
        const int i = e % 3;
        err_out[e] = (e < 3) ? p1[i] - p0[i] - o.lvs : p0[i] - p1[i] - o.lvs;  // (lvs: max_displacement)
      } else {
        const int col = e - 6, k = col / D, j = col % D;
        const double* ab = sm + S.jax + ((o.first + k) * D + j) * 6;
        const double* pk = k ? p1 : p0;
        const bool moves = (o.joint_mask >> j) & 1;
        const double J[3] = {ab[1] * pk[2] - ab[2] * pk[1] - ab[3], ab[2] * pk[0] - ab[0] * pk[2] - ab[4],
                             ab[0] * pk[1] - ab[1] * pk[0] - ab[5]};
        for (int i = 0; i < 3; ++i) {
          const double v = moves ? (k ? J[i] : -J[i]) : 0.0;
          jac_out[i * p.cart_stride + col] = v;
          jac_out[(3 + i) * p.cart_stride + col] = -v;
        }
      }
    }

    // ---- dense candidate collision rows (collision_terms.cpp:203-250, 343-383, 540-556, 655-691) ----
    // candidate r = (collision object k, robot sphere s, obstacle o);  row = {grad[D], dist0, margin, coeff|0}
    // One warp per collision object (= waypoint), one lane per candidate: the lane builds its row in registers and
    // stores it straight to HBM as 16-byte pieces (the L*O rows of an object are contiguous, so a warp fills whole
    // sectors between its stores); the activity mask of 32 candidates is one ballot.  No block barrier inside.
    const int LO = L * O, lane_c = tid & 31;
    const double* obst = sm + S.obst;
    double* rows_out = p.coll_rows + slot * static_cast<size_t>(p.n_coll_cand) * p.coll_stride;
    const float inv_O = 1.0f / static_cast<float>(O);
    for (;;) {
      int k = 0;
      if (lane_c == 0) k = atomicAdd(&misc[2], 1);  // next work item: warps take them as they get free
      k = __shfl_sync(0xffffffffu, k, 0);
      if (k >= ex.n_joint_objs + p.n_coll_objs) break;
      if (k < ex.n_joint_objs) {
        // the value of a joint-space object: the SEQUENTIAL sum of its terms in the reference's order (one lane; a chain
        // of ~T*D dependent additions that runs beside the row writers instead of after them)
        if (lane_c == 0) {
          const DevObj& o = aobjs[ex.joint_obj_idx[k]];
          const double* tb = terms + static_cast<size_t>(k) * 2 * T * D;
          const bool two = o.kind == OBJ_JOINT_INEQ_COST || o.kind == OBJ_JOINT_INEQ_CNT;
          double v = 0.0;
          if (two) for (int w = 0; w < 2 * o.n_steps * D; ++w) v += tb[w];
          else for (int w = 0; w < o.n_steps * D; ++w) v += tb[2 * w];
          sm[S.objv + p.n_coll_objs + k] = v;
        }
        continue;
      }
      k -= ex.n_joint_objs;  // the other items: the collision objects
      const DevObj& co = cobjs[k];
      const int t = co.first;
      const double margin = co.margin, reach = co.margin + co.buffer, coeff = co.coeff;
      double vsum = 0.0;  // exact value of the object: its terms added in candidate order (warp-uniform)
      if (co.kind == OBJ_COLL) {
        const double* AB = sm + S.jax + t * D * 6;
        double* const stage = sm + S.fr + (tid >> 5) * (32 * (D + 3));  // this warp's staging tile (the FK frames are dead by now)
        for (int c00 = 0; c00 < LO; c00 += 64) {
          // Two chunks of 32 candidates per pass: the distance chains (loads, fp64 square root) of the two are independent
          // and overlap; the rest of a chunk (row, staging, stores) follows one chunk after the other on one tile.
          int sl2[2];
          double cx2[2], cy2[2], cz2[2], dx2[2], dy2[2], dz2[2], len2[2], dist2[2];
          bool in2[2], act2[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int cnd = c00 + h * 32 + lane_c;
            const bool in = cnd < LO;
            const int sl = in ? static_cast<int>((static_cast<float>(cnd) + 0.5f) * inv_O) : 0, o = in ? cnd - sl * O : 0;
            const double* c = sm + S.sph + (t * L + sl) * 3;
            const double cx = c[0], cy = c[1], cz = c[2];
            const double4 ob = *reinterpret_cast<const double4*>(obst + o * 4);
            const double dx = ob.x - cx, dy = ob.y - cy, dz = ob.z - cz;
            const double len = sqrt(dx * dx + dy * dy + dz * dz);
            const double dist = len - sm[S.sphr + sl] - ob.w;
            sl2[h] = sl; in2[h] = in;
            cx2[h] = cx; cy2[h] = cy; cz2[h] = cz;
            dx2[h] = dx; dy2[h] = dy; dz2[h] = dz;
            len2[h] = len; dist2[h] = dist;
            act2[h] = in && !(dist > reach);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c0 = c00 + h * 32;
            if (c0 < LO) {  // (warp-uniform)
            const int cnd = c0 + lane_c, sl = sl2[h];
            const bool in = in2[h], active = act2[h];
            const double dist = dist2[h];
            double row[D + 3 + ((D + 3) & 1)];
#pragma unroll
            for (int j = 0; j < D; ++j) row[j] = 0.0;
            // The gradient exists only for contacts inside margin + buffer (the reference never builds an expression
            // for a filtered contact, collision_terms.cpp:655-691): the other candidates keep a zero gradient.
            if (active) {
              const double cx = cx2[h], cy = cy2[h], cz = cz2[h];
              const double inv = 1.0 / len2[h];
              const double nx = dx2[h] * inv, ny = dy2[h] * inv, nz = dz2[h] * inv;  // from the robot sphere towards the obstacle
              const double mx = cy * nz - cz * ny, my = cz * nx - cx * nz, mz = cx * ny - cy * nx;  // c x n
              const unsigned jm = ex.sphere_jmask[sl];
#pragma unroll
              for (int j = 0; j < D; ++j) {
                const double2 a01 = *reinterpret_cast<const double2*>(AB + j * 6);
                const double2 a2b0 = *reinterpret_cast<const double2*>(AB + j * 6 + 2);
                const double2 b12 = *reinterpret_cast<const double2*>(AB + j * 6 + 4);
                // d(dist)/dq_j = -n . d(c)/dq_j = B_j . n - A_j . (c x n)
                const double g = (a2b0.y * nx + b12.x * ny + b12.y * nz) - (a01.x * mx + a01.y * my + a2b0.x * mz);
                row[j] = ((jm >> j) & 1u) ? g : 0.0;
              }
            }
            row[D] = dist;
            row[D + 1] = margin;
            row[D + 2] = active ? coeff : 0.0;
            if constexpr (((D + 3) & 1) == 0) {
              // rows are 16-byte aligned (D + 3 even, 256-byte aligned buffers): the 32 rows of the chunk are staged in
              // shared memory and leave as warp-contiguous 16-byte stores (512 contiguous bytes per store instruction,
              // 2.5 KB contiguous per chunk).  (A cp.async.bulk store of the tile moves the same bytes, but the tile can
              // only be refilled once the bulk engine has read it, which serialises the row phase; plain stores are fire
              // and forget.)
              if (in) {
                double2* d2 = reinterpret_cast<double2*>(stage + lane_c * (D + 3));
#pragma unroll
                for (int i = 0; i < (D + 3) / 2; ++i) d2[i] = make_double2(row[2 * i], row[2 * i + 1]);
              }
              __syncwarp();
              {
                const int nrows = (LO - c0 < 32) ? LO - c0 : 32;
                const double2* src2 = reinterpret_cast<const double2*>(stage);
                double2* dst2 = reinterpret_cast<double2*>(rows_out + static_cast<size_t>(co.src_off + c0) * (D + 3));
                const int n2 = nrows * ((D + 3) / 2);
#pragma unroll
                for (int i = 0; i < (D + 3) / 2; ++i) {
                  const int e = i * 32 + lane_c;
                  if (e < n2) dst2[e] = src2[e];
                }
              }
              __syncwarp();  // the tile may be refilled
            } else if (in) {
              double* dstp = rows_out + static_cast<size_t>(co.src_off + cnd) * (D + 3);
#pragma unroll
              for (int i = 0; i < D + 3; ++i) dstp[i] = row[i];
            }
            const unsigned bal = __ballot_sync(0xffffffffu, active);
            if (lane_c == 0 && bal) atomicOr(&mask[k * p.coll_words + (c0 >> 6)], static_cast<unsigned long long>(bal) << (c0 & 63));
            const double mine = active ? fmax(margin - dist, 0.0) * coeff : 0.0;
            unsigned nzb = __ballot_sync(0xffffffffu, mine != 0.0);
            while (nzb) {  // warp-uniform: the non-zero terms in candidate order (zeros do not change the sum)
              vsum += __shfl_sync(0xffffffffu, mine, __ffs(nzb) - 1);
              nzb &= nzb - 1;
            }
            }
          }
        }
      } else {
        // ---- continuous ("cast") collision of the step pair (t, t+1): collision_terms.cpp:262-323, 468-538,
        // 1071-1173 with the closed-form swept sphere (capsule) of SURVEY.md section 8d; the same rules as the oracle's
        // CastCollisionEval.  The sub-trajectory is as long as the reference's (nsub = ceil(|q1 - q0| / lvs), unbounded,
        // :1118-1155).  Pass 1 walks the sub-segments one after the other (one warp FK per interior state, the centres of
        // the two ends of the running sub-segment in shared memory) and lists the ACTIVE contacts (sphere, obstacle,
        // sub-segment).  Pass 2 ranks them in the reference's order (link pair, then sub-segment) and writes one row
        // {g0[D], g1[D], dist, margin, coeff} per contact into slot `rank` of the pair's row block; the mask of the pair
        // has its low `count` bits set, so the QP step picks the rows up like any other active candidates.  The gradients
        // need FKs per ACTIVE contact only (both ends of its sub-segment and its contact-time state).
        const int CAP = ex.cast_cap, CS = 2 * D + 3;
        // LVS_DISCRETE (DiscreteCollisionEvaluator, collision_terms.cpp:744-893): the same machinery with a discrete test
        // at each of the nsub + 1 STATES of the sub-trajectory (a sub-segment of zero length: s = 0, cc_time = i / nsub,
        // Time0 | Time1 at the waypoints, one link frame for both reference points).
        const bool sfix = co.cast_flags & CAST_START_FIXED, efix = co.cast_flags & CAST_END_FIXED, disc = co.cast_flags & CAST_LVS_DISCRETE;
        const double* q0 = xs + t * D;
        const double* q1 = q0 + D;
        double d2 = 0.0;
#pragma unroll
        for (int j = 0; j < D; ++j) d2 += (q1[j] - q0[j]) * (q1[j] - q0[j]);
        const double qd = sqrt(d2);
        int nsub = 1;
        bool overflow = false;
        if (qd > co.lvs) {
          const double nn = ceil(qd / co.lvs);
          overflow = nn > 32767.0;  // (the contact key holds the sub-segment in 15 bits)
          nsub = overflow ? 32767 : static_cast<int>(nn);
        }
        double* F = sm + S.wscr + (tid >> 5) * S.wscr_stride;  // frames of one state
        double* cenA = F + p.S * 12;                            // [L][3] sphere centres at the start of the sub-segment
        double* cenB = cenA + L * 3;                            // ... and at its end
        double* qv = cenB + L * 3 + (L & 1);
        // the contacts of this pair (written and read by this warp only; volatile: no stale L1 lines, no reordering)
        volatile double* csd = ex.cast_scratch + (static_cast<size_t>(blockIdx.x) * (kEvalThreads / 32) + (tid >> 5)) * 4 * CAP;  // [CAP][2]: s, distance
        volatile int* ckey = reinterpret_cast<volatile int*>(csd + 2 * CAP);  // [CAP] (sphere * O + obstacle) << 15 | sub-segment
        volatile int* crank = ckey + CAP;                                     // [CAP]
        volatile double* cval = csd + 3 * CAP;                                // [CAP] hinge values in canonical order
        // centres of every sphere at the state `frac` of the way from q0 to q1 (i = 0 / nsub: the waypoints themselves)
        auto centres_at = [&](int i, double* dstc) {
          if (i == 0 || i == nsub) {
            const double* src = sm + S.sph + ((i == 0 ? t : t + 1) * L) * 3;
            for (int w = lane_c; w < L * 3; w += 32) dstc[w] = src[w];
          } else {
            if (lane_c < D) qv[lane_c] = q0[lane_c] + (q1[lane_c] - q0[lane_c]) * (static_cast<double>(i) / nsub);
            __syncwarp();
            warp_fk(p, qv, F, lane_c);
            for (int w = lane_c; w < L; w += 32) {
              const DevSphere& sp = sphs[w];
              const double* f = F + sp.segment * 12;
              for (int a = 0; a < 3; ++a)
                dstc[w * 3 + a] = f[a * 3] * sp.c[0] + f[a * 3 + 1] * sp.c[1] + f[a * 3 + 2] * sp.c[2] + f[9 + a];
            }
          }
          __syncwarp();
        };
        int count = 0;
        centres_at(0, cenA);
        const int n_slots = disc ? nsub + 1 : nsub;
        for (int i = 0; i < n_slots; ++i) {
          if (!disc) centres_at(i + 1, cenB);
          else if (i > 0) centres_at(i, cenA);
          for (int c0 = 0; c0 < LO; c0 += 32) {
            const int pr = c0 + lane_c;
            const bool in = pr < LO;
            const int sl = in ? static_cast<int>((static_cast<float>(pr) + 0.5f) * inv_O) : 0, o = in ? pr - sl * O : 0;
            const double* ca = cenA + sl * 3;
            const double* cb = (disc ? cenA : cenB) + sl * 3;
            const double4 ob = *reinterpret_cast<const double4*>(obst + o * 4);
            const double wx = cb[0] - ca[0], wy = cb[1] - ca[1], wz = cb[2] - ca[2];
            const double ww = wx * wx + wy * wy + wz * wz;
            const double wd = (ob.x - ca[0]) * wx + (ob.y - ca[1]) * wy + (ob.z - ca[2]) * wz;
            double sc = (ww > 0.0) ? wd / ww : 0.0;
            sc = sc < 0.0 ? 0.0 : (sc > 1.0 ? 1.0 : sc);
            const double dx = ob.x - (ca[0] + sc * wx), dy = ob.y - (ca[1] + sc * wy), dz = ob.z - (ca[2] + sc * wz);
            const double len = sqrt(dx * dx + dy * dy + dz * dz);
            const double dist = len - sm[S.sphr + sl] - ob.w;
            const bool time0 = (i == 0 && sc == 0.0), time1 = disc ? (i == nsub) : (i == nsub - 1 && sc == 1.0);
            const bool active = in && !(dist > reach) && !(sfix && time0) && !(efix && time1);
            const unsigned bal = __ballot_sync(0xffffffffu, active);
            const int pos = count + __popc(bal & ((1u << lane_c) - 1u));
            if (active && pos < CAP) {
              csd[2 * pos] = sc;
              csd[2 * pos + 1] = dist;
              ckey[pos] = (pr << 15) | i;
            }
            count += __popc(bal);
          }
          __syncwarp();
          if (!disc)
            for (int w = lane_c; w < L * 3; w += 32) cenA[w] = cenB[w];  // the end of this sub-segment starts the next
          __syncwarp();
        }
        if (count > CAP) {
          overflow = true;
          count = CAP;
        }
        if (overflow && lane_c == 0) p.lvs_overflow[b] = 1;
        // ranks in the reference's order: link pair (sphere, obstacle) first, then the sub-segment (keys are unique)
        for (int c = lane_c; c < count; c += 32) {
          const int key = ckey[c];
          int r = 0;
          for (int c2 = 0; c2 < count; ++c2) r += ckey[c2] < key;
          crank[c] = r;
          cval[r] = fmax(margin - csd[2 * c + 1], 0.0) * coeff;
        }
        __syncwarp();
        for (int c = 0; c < count; ++c) {  // warp-uniform loop over the active contacts
          const int key = ckey[c], i_s = key & 32767, pr_s = key >> 15;
          const int sl_s = static_cast<int>((static_cast<float>(pr_s) + 0.5f) * inv_O), o_s = pr_s - sl_s * O;
          const double sc = csd[2 * c], dist = csd[2 * c + 1];
          const DevSphere& sp = sphs[sl_s];
          // centre and offset (centre - link origin = R_link * c_local) of the sphere at both ends of its sub-segment
          double ca[3], cb[3], offa[3], offb[3];
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const int st = disc ? i_s : i_s + kk;
            double* cc3 = kk ? cb : ca;
            double* of3 = kk ? offb : offa;
            if (st == 0 || st == nsub) {
              const int wp = (st == 0) ? t : t + 1;
#pragma unroll
              for (int a = 0; a < 3; ++a) {
                cc3[a] = sm[S.sph + (wp * L + sl_s) * 3 + a];
                of3[a] = sm[S.spo + (wp * L + sl_s) * 3 + a];
              }
            } else {
              if (lane_c < D) qv[lane_c] = q0[lane_c] + (q1[lane_c] - q0[lane_c]) * (static_cast<double>(st) / nsub);
              __syncwarp();
              warp_fk(p, qv, F, lane_c);
              const double* f = F + sp.segment * 12;
#pragma unroll
              for (int a = 0; a < 3; ++a) {
                const double off = f[a * 3] * sp.c[0] + f[a * 3 + 1] * sp.c[1] + f[a * 3 + 2] * sp.c[2];
                of3[a] = off;
                cc3[a] = off + f[9 + a];
              }
              __syncwarp();
            }
          }
          const double4 ob = *reinterpret_cast<const double4*>(obst + o_s * 4);
          const double wx = cb[0] - ca[0], wy = cb[1] - ca[1], wz = cb[2] - ca[2];
          const double dx = ob.x - (ca[0] + sc * wx), dy = ob.y - (ca[1] + sc * wy), dz = ob.z - (ca[2] + sc * wz);
          const double len = sqrt(dx * dx + dy * dy + dz * dz);
          const double nxs = dx / len, nys = dy / len, nzs = dz / len;
          const double cc_s = (i_s + sc) / nsub;
          if (lane_c < D) qv[lane_c] = (cc_s == 1.0) ? q1[lane_c] : q0[lane_c] + (q1[lane_c] - q0[lane_c]) * cc_s;
          __syncwarp();
          warp_fk(p, qv, F, lane_c);  // Jacobian at the contact-time state (GetGradient, :276-285)
          double* rowp = rows_out + static_cast<size_t>(co.src_off + crank[c]) * CS;
          if (lane_c < D) {
            const int j = lane_c, sg = ex.joint_seg[j];
            const DevSegment& g = segs[sg];
            const double* f = F + sg * 12;
            const double* pl = F + sp.segment * 12 + 9;
            const double ax = f[0] * g.axis[0] + f[1] * g.axis[1] + f[2] * g.axis[2];
            const double ay = f[3] * g.axis[0] + f[4] * g.axis[1] + f[5] * g.axis[2];
            const double az = f[6] * g.axis[0] + f[7] * g.axis[1] + f[8] * g.axis[2];
            const bool moves = (ex.sphere_jmask[sl_s] >> j) & 1u, rev = g.joint_type == 1;
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
              double gg = 0.0;
              if (!((kk == 0 && sfix) || (kk == 1 && efix))) {  // a fixed side contributes nothing
                // reference point: link origin at the contact-time state + R_link(sub-segment start | end) * c_local
                const double* off = kk ? offb : offa;
                const double rx = pl[0] + off[0] - f[9], ry = pl[1] + off[1] - f[10], rz = pl[2] + off[2] - f[11];
                const double jx = rev ? ay * rz - az * ry : ax, jy = rev ? az * rx - ax * rz : ay,
                             jz = rev ? ax * ry - ay * rx : az;
                gg = -(nxs * jx + nys * jy + nzs * jz) * (kk == 0 ? 1.0 - cc_s : cc_s);
              }
              rowp[kk * D + j] = moves ? gg : 0.0;
            }
          }
          if (lane_c == 0) {
            rowp[2 * D] = dist;
            rowp[2 * D + 1] = margin;
            rowp[2 * D + 2] = coeff;
          }
          __syncwarp();
        }
        // the pair's mask: its first `count` row slots are active; its exact value: the hinge terms in canonical order
        for (int w = lane_c; w < p.coll_words; w += 32) {
          const int lo = w * 64;
          mask[k * p.coll_words + w] = (count >= lo + 64) ? ~0ull : ((count > lo) ? ((1ull << (count - lo)) - 1ull) : 0ull);
        }
        if (lane_c == 0)
          for (int c = 0; c < count; ++c) vsum += cval[c];
      }
      if (lane_c == 0) sm[S.objv + k] = vsum;
    }
    // ---- AvoidSingularity rows: a warp per object, as its collision work runs out ----
    if constexpr (SING != 0)
      singularity_objects<D>(ex, xs, segs, sm + S.sing, p.cart_err + slot * p.n_cart_rows,
                             p.cart_jac + slot * p.n_cart_rows * p.cart_stride, p.cart_stride);
    __syncthreads();
    EVAL_PROF(5);
    for (int i = tid; i < n_mask_words; i += kEvalThreads) p.coll_mask[slot * n_mask_words + i] = mask[i];
  }

  // ---- exact values at the evaluated point (Cost::value / Constraint::violation) -------------------
  // Every object's value is the SEQUENTIAL sum of its terms in the reference's order (the merit decisions compare
  // such sums), so the terms are produced in parallel and one lane adds them up in order: joint-space objects
  // from the term buffer, collision objects by walking the non-zero candidates of the warp in lane order.
  double* out_cost = (mode == EVAL_ONLY) ? p.cost_vals + static_cast<size_t>(b) * p.n_costs
                                         : (mode == EVAL_INIT ? p.cost_vals : p.new_cost_vals) + static_cast<size_t>(b) * p.n_costs;
  double* out_viol = (mode == EVAL_ONLY) ? p.cnt_viols + static_cast<size_t>(b) * p.n_cnts
                                         : (mode == EVAL_INIT ? p.cnt_viols : p.new_cnt_viols) + static_cast<size_t>(b) * p.n_cnts;
  if (!qp_failed) {
    // (the barrier after the row phase covers everything read here: the in-order sums in shared memory and the
    // cart_err rows this CTA wrote to global memory)
    const int n_obj = p.n_costs + p.n_cnts;
    EVAL_PROF(6);
    for (int i = tid; i < n_obj; i += kEvalThreads) {  // one thread per object
      const bool is_cnt = i >= p.n_costs;
      const DevObj& o = aobjs[i];
      double v = 0.0;
      if (o.kind <= OBJ_JOINT_INEQ_CNT) {
        int slot_j = 0;
        for (int k = 0; k < ex.n_joint_objs; ++k) slot_j = (ex.joint_obj_idx[k] == i) ? k : slot_j;
        v = sm[S.objv + p.n_coll_objs + slot_j];  // summed in order by a warp of the row phase
      } else if (o.kind == OBJ_CART_POSE) {
        const double* e = p.cart_err + slot * p.n_cart_rows + o.src_off;
        for (int r = 0; r < o.n_rows; ++r) v += fabs(e[r]);
      } else if (o.kind == OBJ_CART_VEL) {
        const double* e = p.cart_err + slot * p.n_cart_rows + o.src_off;
        for (int r = 0; r < 6; ++r) v += is_cnt ? fmax(e[r], 0.0) : fabs(e[r]);  // INEQ violation | ABS cost
      } else if (SING != 0 && o.kind == OBJ_SINGULARITY) {
        const double e = p.cart_err[slot * p.n_cart_rows + o.src_off];
        v = is_cnt ? fmax(e, 0.0) : fabs(e);  // INEQ violation | ABS cost
      } else {
        v = sm[S.objv + o.kernel_slot];  // collision object: summed by the warp that built its rows
      }
      if (is_cnt) out_viol[i - p.n_costs] = v;
      else out_cost[i] = v;
    }
  }
  EVAL_PROF(7);
  EVAL_PROF_END();
  if (mode == EVAL_ONLY) return;  // tb200_convexify_batch: exact values only, no SQP state touched
  __threadfence_block();
  __syncthreads();

  // ---- SQP iteration log (DESIGN.md section 4.7; off: one uniform branch) ----------------------------
  // One record for the initial evaluation and one for every QP solve (the places n_qp_solves counts).  Everything but the
  // decision's outcome goes out here, before the decision, because the penalty step below inflates the merit
  // coefficients this decision used; thread 0 adds the merits, the action and the end status in the decision and only
  // then counts the record (so the state machine keeps no log values live).  A failed QP has no model, point or values:
  // NaN.
  if (ex.log != nullptr) {
    log_record_arrays(p, ex, mode, b, qp_failed, aobjs, out_cost, out_viol, xs);
    __syncthreads();
  }

  // ---- trust-region / penalty state machine (thread 0), optimizers.cpp:811-968 ----------------------
  if (tid == 0) {
    const SqpParams& sp = ex.sqp[b];  // (this trajectory's row)
    double* mu = p.merit_coeffs + static_cast<size_t>(b) * p.n_cnts;
    double* cv = p.cost_vals + static_cast<size_t>(b) * p.n_costs;
    double* kv = p.cnt_viols + static_cast<size_t>(b) * p.n_cnts;
    double trust = p.trust[b];
    int accept = 0, finished = 0, status = 5;
    int top = 0;  // the next QP begins a new SQP iteration (iter = 1 of a merit round, or ++iter): the time-limit check
    enum { NEXT_QP = 0, AFTER_LOOP = 1, PENALTY = 2 } go = NEXT_QP;
    if (ex.cast && p.lvs_overflow[b]) {
      // a step pair needed more LVS sub-segments than the candidate layout holds: the trajectory stops here and
      // tb200_solve_batch reports TB200_ERR_UNSUPPORTED (the layout is never truncated silently)
      status = 4;  // OPT_FAILED
      finished = 1;
    } else if (mode == EVAL_INIT) {
      p.n_func_evals[b] = 1;
      accept = 2;  // rows of buffer 0 are the rows at x
      top = 1;
    } else {
      p.n_qp_solves[b] += 1;
      double tr_old = 0, tr_model = 0, tr_new = 0;
      int tr_action = 3;
      const double tr_trust = trust;
      if (qp_failed) {  // failure ladder, optimizers.cpp:817-842
        int f = p.qp_failures[b];
        if (f < sp.max_qp_solver_failures - 1) {
          trust *= sp.trust_shrink_ratio;
          p.qp_failures[b] = f + 1;
          go = (trust >= sp.min_trust_box_size) ? NEXT_QP : AFTER_LOOP;
        } else if (f == sp.max_qp_solver_failures - 1) {
          trust = sp.min_trust_box_size;
          p.qp_failures[b] = f + 1;
          go = (trust >= sp.min_trust_box_size) ? NEXT_QP : AFTER_LOOP;
        } else {
          status = 4;  // OPT_FAILED
          finished = 1;
        }
      } else {
        p.n_func_evals[b] += 1;
        const double* mc = p.model_cost_vals + static_cast<size_t>(b) * p.n_costs;
        const double* mk = p.model_cnt_viols + static_cast<size_t>(b) * p.n_cnts;
        double old_merit = 0, model_merit = 0, new_merit = 0, s;
        s = 0; for (int i = 0; i < p.n_costs; ++i) s += cv[i];
        old_merit = s;
        s = 0; for (int i = 0; i < p.n_cnts; ++i) s += kv[i] * mu[i];
        old_merit += s;
        s = 0;
        for (int i = 0; i < p.n_costs; ++i)  // quadratic joint costs are their own convex model
          s += (p.cost_objs[i].kind == OBJ_JOINT_EQ_COST) ? out_cost[i] : mc[i];
        model_merit = s;
        s = 0; for (int i = 0; i < p.n_cnts; ++i) s += mk[i] * mu[i];
        model_merit += s;
        s = 0; for (int i = 0; i < p.n_costs; ++i) s += out_cost[i];
        new_merit = s;
        s = 0; for (int i = 0; i < p.n_cnts; ++i) s += out_viol[i] * mu[i];
        new_merit += s;
        const double approx = old_merit - model_merit, exact = old_merit - new_merit, ratio = exact / approx;
        tr_old = old_merit; tr_model = model_merit; tr_new = new_merit;
        if (approx < sp.min_approx_improve) { go = PENALTY; tr_action = 2; }
        else if (approx / old_merit < sp.min_approx_improve_frac) { go = PENALTY; tr_action = 2; }
        else if (exact < 0 || ratio < sp.improve_ratio_threshold) {
          trust *= sp.trust_shrink_ratio;
          go = (trust >= sp.min_trust_box_size) ? NEXT_QP : AFTER_LOOP;
          tr_action = 0;
        } else {
          accept = 1;
          trust *= sp.trust_expand_ratio;
          go = AFTER_LOOP;
          tr_action = 1;
        }
      }
      if (p.trace && p.trace_len[b] < p.trace_cap) {
        double* te = p.trace + (static_cast<size_t>(b) * p.trace_cap + p.trace_len[b]) * 14;
        te[0] = p.merit_round[b]; te[1] = p.sqp_iter[b]; te[2] = tr_trust; te[3] = tr_old; te[4] = tr_model; te[5] = tr_new;
        const double* g = p.dbg + static_cast<size_t>(b) * 16;
        te[6] = g[0]; te[7] = g[1]; te[8] = tr_action; te[9] = g[4]; te[10] = g[5]; te[11] = g[3]; te[12] = g[2]; te[13] = g[14];
        p.trace_len[b] += 1;
      }
      if (ex.log != nullptr && ex.log_len[b] < ex.log_cap) {  // (the merits stay NaN for a failed QP)
        double* lh = ex.log + (static_cast<size_t>(b) * ex.log_cap + ex.log_len[b]) * ex.log_stride;
        if (!qp_failed) { lh[LOG_OLD_MERIT] = tr_old; lh[LOG_MODEL_MERIT] = tr_model; lh[LOG_NEW_MERIT] = tr_new; }
        lh[LOG_ACTION] = tr_action;
      }
      if (!finished && go == AFTER_LOOP) {
        const double* kk = accept ? out_viol : kv;
        if (trust < sp.min_trust_box_size) go = PENALTY;
        else if (p.sqp_iter[b] >= sp.max_iter) {
          double mx = -1e300;
          for (int i = 0; i < p.n_cnts; ++i) mx = fmax(mx, kk[i]);
          status = (p.n_cnts == 0 || mx < sp.cnt_tolerance) ? 0 : 1;
          finished = 1;
        } else {
          p.sqp_iter[b] += 1;
          p.qp_failures[b] = 0;
          go = NEXT_QP;
          top = 1;
        }
      }
      if (!finished && go == PENALTY) {  // optimizers.cpp:938-968
        const double* kk = accept ? out_viol : kv;
        double mx = -1e300;
        for (int i = 0; i < p.n_cnts; ++i) mx = fmax(mx, kk[i]);
        if (p.n_cnts == 0 || mx < sp.cnt_tolerance) {
          status = 0;
          finished = 1;
        } else {
          for (int i = 0; i < p.n_cnts; ++i)
            if (!sp.inflate_constraints_individually || kk[i] > sp.cnt_tolerance) mu[i] *= sp.merit_coeff_increase_ratio;
          trust = fmax(trust, sp.min_trust_box_size / sp.trust_shrink_ratio * 1.5);
          const int round = p.merit_round[b] + 1;
          p.merit_round[b] = round;
          if (round >= sp.max_merit_coeff_increases) {
            status = 2;  // OPT_PENALTY_ITERATION_LIMIT
            finished = 1;
          } else {
            p.sqp_iter[b] = 1;
            p.qp_failures[b] = 0;
            top = 1;
          }
        }
      }
    }
    if (ex.log != nullptr && (mode == EVAL_INIT || !(ex.cast && p.lvs_overflow[b]))) {  // the record is complete
      const int n = ex.log_len[b];
      if (n < ex.log_cap) {
        ex.log[(static_cast<size_t>(b) * ex.log_cap + n) * ex.log_stride + LOG_ENDED] = finished ? status : -1;
        ex.log_len[b] = n + 1;
      } else {
        ex.log_dropped[b] += 1;
      }
    }
    p.trust[b] = trust;
    p.sqp_top[b] = top;  // (0 on a trust-region or QP-failure retry: no check inside the inner loop)
    if (mode == EVAL_STEP) p.qp_done[b] = 0;
    misc[0] = accept;
    if (finished) {
      misc[1] = 1;
      p.status[b] = status;
      if (status == 0 && p.group_stop) {  // release: the siblings read the flag at their next iteration top (solve_kernel.cuh)
        __threadfence();
        atomicExch(p.group_done + b / p.group_size, 1);
      }
      atomicSub(p.active_count, 1);
    } else {
      misc[1] = 0;
    }
  }
  __syncthreads();
  const int accept = misc[0];
  if (accept) {  // results_.x = new_x, cost_vals / cnt_viols = new values (optimizers.cpp:906-909)
    double* xd = p.x + static_cast<size_t>(b) * N;
    for (int i = tid; i < N; i += kEvalThreads) xd[i] = xs[i];
    if (accept == 1) {
      for (int i = tid; i < p.n_costs; i += kEvalThreads) p.cost_vals[static_cast<size_t>(b) * p.n_costs + i] = out_cost[i];
      for (int i = tid; i < p.n_cnts; i += kEvalThreads) p.cnt_viols[static_cast<size_t>(b) * p.n_cnts + i] = out_viol[i];
    }
    if (tid == 0) p.cur_buf[b] = dst;
  }
}

// The evaluation step as a function of its own (the persistent SQP kernel calls it beside its QP step; the stand-alone
// kernel below inlines the implementation).
template <int DD, int SING = 0>
__device__ __noinline__ void eval_step(const DevProblem& p, const EvalExtra& ex, const int mode, const int b,
                                       const double* x_in /*EVAL_ONLY*/) {
  bool tables_ready = false;  // (the QP step used the same shared memory in between)
  eval_step_impl<DD, SING>(p, ex, mode, b, x_in, tables_ready);
}

// Two CTAs per SM cap the 7-joint instance at 128 registers, and on sm_90a ptxas spills a few of them; one CTA per SM
// needs 180 and none spill.  Measured on an H100 (configs[2], full batch of 1024): 111-119 us per launch with two
// CTAs per SM against 140-144 us with one, the same SQP throughput either way.  So two stay.
#ifndef TB200_EVAL_MIN_BLOCKS
#define TB200_EVAL_MIN_BLOCKS 2
#endif
// Stand-alone launch, one CTA per trajectory: the initial evaluation of a solve (EVAL_INIT) and the kernel-level
// convexify entry point (EVAL_ONLY).  Inside a solve the same code runs as a step of solve_kernel.cuh.
template <int DD, int SING = 0>
__global__ void __launch_bounds__(kEvalThreads, (DD <= 8) ? TB200_EVAL_MIN_BLOCKS : 2)
eval_convexify_decide_kernel(const __grid_constant__ DevProblem p, const __grid_constant__ EvalExtra ex, int mode,
                             const double* x_in /*EVAL_ONLY*/) {
  // persistent CTAs: the grid fills the SMs once and every CTA takes the next trajectory when it is done with one
  // (1024 trajectories over 132 SMs x 2 resident CTAs: no tail wave of half-empty SMs)
  __shared__ int s_next;
  bool tables_ready = false;  // the robot / object tables stay in shared memory from one trajectory to the next
  for (;;) {
    if (threadIdx.x == 0) s_next = atomicAdd(ex.work_counter, 1);
    __syncthreads();
    const int b = s_next;
    __syncthreads();
    if (b >= p.B) return;
    eval_step_impl<DD, SING>(p, ex, mode, b, x_in, tables_ready);
    __syncthreads();
  }
}

}  // namespace tb200
