// Device-side data model of the batched SQP hot path (sm_90a).  See DESIGN.md §3 for the HBM layout.
#pragma once
#include <cstddef>
#include <cstdint>

namespace tb200 {

constexpr int kMaxDof = 16;
constexpr int kMaxSeg = 40;
constexpr int kMaxSpheres = 32;
constexpr int kMaxSteps = 64;

struct DevSegment {
  int parent, joint_type, q_index, pad;
  double R[9];  // origin rotation, row-major
  double p[3];
  double axis[3];
};
struct DevSphere {
  int segment, pad;
  double c[3];
  double r;
};

// One sco::Cost / sco::Constraint object as hatched by the reference's TermInfo::hatch
// (trajopt/src/problem_description.cpp), in OptProb order (constraints: EQ first, then INEQ).
enum ObjKind {
  OBJ_JOINT_EQ_COST = 0,   // JointPos/Vel/AccEqCost       trajectory_costs.cpp:12-138, 257-301, 502-549
  OBJ_JOINT_INEQ_COST = 1, // Joint*IneqCost               trajectory_costs.cpp:303-374
  OBJ_JOINT_EQ_CNT = 2,    // Joint*EqConstraint           trajectory_costs.cpp:139-183
  OBJ_JOINT_INEQ_CNT = 3,  // Joint*IneqConstraint         trajectory_costs.cpp:185-254
  OBJ_CART_POSE = 4,       // CartPose ABS cost / EQ cnt   kinematic_terms.cpp:187-366
  OBJ_COLL = 5,            // discrete collision per step  collision_terms.cpp:1283-1412
  OBJ_CART_VEL = 6,        // CartVel per step pair        kinematic_terms.cpp:368-425, problem_description.cpp:1011-1057
  OBJ_COLL_CAST = 7,       // continuous (cast) collision per step pair  collision_terms.cpp:262-323, 468-538, 1071-1173
  OBJ_SINGULARITY = 8      // AvoidSingularity per step: ABS cost / INEQ cnt  kinematic_terms.cpp:586-642
};
struct DevObj {
  int kind;
  int is_cnt;     // 0 cost, 1 constraint
  int order;      // joint stencil order 0/1/2
  int first;      // first stencil row (joint) / timestep (cart, collision)
  int n_steps;    // joint: number of stencil rows in time
  int term;       // index into the joint parameter table / cart table
  int src_off;    // cart: first row in the cart buffers; collision: first candidate
  int n_rows;     // cart: rows; collision: candidates (n_spheres * n_obstacles); joint: rows emitted
  int link;       // cart: segment
  union {
    int target_slot;  // cart_pose: static target in cart_targets[b] (-1: the term's own target_pose)
    int kernel_slot;  // collision: position in the kernel order (coll_objs), where the evaluation kernel leaves its value
  };
  int list_index;  // cart, vel and coll tables: index of the object in cost_objs (cost) or cnt_objs (constraint)
  union {
    int joint_mask;  // cart_vel: joints moving the link (bit mask)
    int cast_flags;  // cast collision: CAST_START_FIXED, CAST_END_FIXED, CAST_LVS_DISCRETE
  };
  double coeff, margin, buffer;  // avoid_singularity: coeff = the term's coefficient, margin = its lambda
  // cast collision: longest valid segment length (max double: never subdivide); cart_vel: max_displacement.  (One
  // name: unlike the int unions above, a union of the two doubles changes the evaluation kernel's instructions.)
  double lvs;
};
enum CastFlag { CAST_START_FIXED = 1, CAST_END_FIXED = 2, CAST_LVS_DISCRETE = 4 };  // DevObj::cast_flags
// the evaluation kernel copies the collision objects to shared memory as raw doubles
static_assert(sizeof(DevObj) == 80, "DevObj layout");
static_assert(offsetof(DevObj, coeff) == 48 && offsetof(DevObj, margin) == 56 && offsetof(DevObj, buffer) == 64 &&
                  offsetof(DevObj, lvs) == 72,
              "DevObj layout");
struct DevJointTerm {
  double coeffs[kMaxDof], targets[kMaxDof], upper[kMaxDof], lower[kMaxDof];
};
struct DevCartTerm {
  double src_R[9], src_p[3];  // source_frame_offset
  double tgt[7];              // default static target (xyz + wxyz)
  int idx[6];                 // kept error components
  double coeff[6];
  int n_idx, pad;
};

enum RowInt { RI_BASE = 0, RI_CNT, RI_STRIDE, RI_AUX, RI_OBJ, RI_PAD, RI_NINTS };
enum AuxKind { AUX_NONE = 0, AUX_HINGE = 1, AUX_ABS = 2 };

struct QpSettings {
  double rho, sigma, alpha, eps_abs, eps_rel, eps_prim_inf, eps_dual_inf, delta, adaptive_rho_tolerance;
  int max_iter, scaling, check_termination, adaptive_rho, adaptive_rho_interval, polishing, polish_refine_iter,
      warm_starting, early_polish_every, early_polish_from;
};
struct SqpParams {
  double improve_ratio_threshold, min_trust_box_size, min_approx_improve, min_approx_improve_frac;
  double trust_shrink_ratio, trust_expand_ratio, cnt_tolerance, max_merit_coeff_increases;
  double merit_coeff_increase_ratio, initial_merit_error_coeff, trust_box_size;
  int max_iter, max_qp_solver_failures, inflate_constraints_individually, pad;
  double max_time;  // seconds; checked at the top of an SQP iteration (solve_kernel.cuh), DBL_MAX: no limit
};

// Everything a kernel needs; passed by value (pointers into device memory).
struct DevProblem {
  int B, T, D, N, HB;          // batch, steps, dof, T*D, half bandwidth (2*D)
  int S, L, O, obstacles_per_traj;
  int n_costs, n_cnts, n_cart_rows, cart_stride, n_coll_cand, coll_stride;
  int n_cart_targets, n_fixed, max_rows, row_stride, coll_words;  // coll_words: 64-bit mask words per collision object
  int n_sparse_lists, n_band;  // n_band: band offsets k with a structurally non-zero P(i, i-k)
  int band_offs[32];           // those offsets, ascending (joint costs: 0, D, 2D)
  const DevSegment* segs;
  const DevSphere* spheres;
  const double* lower;
  const double* upper;
  const DevObj* cost_objs;
  const DevObj* cnt_objs;
  const DevJointTerm* joint_terms;
  const DevCartTerm* cart_terms;
  const int* fixed_vars;       // [n_fixed]
  const double* Pband;         // [N][HB+1]  P(i, i-k), objective Hessian of the state-independent quadratic costs
  const double* qlin;          // [N]
  // per-trajectory inputs
  const double* init_traj;     // [B][N]
  const double* cart_targets;  // [B][n_cart_targets][7]
  const double* obstacles;     // [B or 1][O][4]
  // SQP state (per trajectory)
  double* x;                   // [B][N] current iterate
  double* new_x;               // [B][N] QP solution (trajectory part)
  double* trust;               // [B]
  double* merit_coeffs;        // [B][n_cnts]
  double* cost_vals;           // [B][n_costs]   exact at x
  double* cnt_viols;           // [B][n_cnts]
  double* new_cost_vals;       // exact at new_x
  double* new_cnt_viols;
  double* model_cost_vals;     // [B][n_costs]   (row based costs only; quadratic costs are exact)
  double* model_cnt_viols;     // [B][n_cnts]
  int* status;                 // [B] OptStatus, TB200_OPT_INVALID while running
  int* sqp_iter;               // [B]
  int* merit_round;            // [B]
  int* qp_failures;            // [B]
  int* qp_status;              // [B] CvxOptStatus of the last QP
  int* cur_buf;                // [B] which convexification buffer holds the rows at x
  int* n_qp_solves;
  int* n_func_evals;
  int* n_admm_iters;
  int* active_count;           // [1]
  // convexification buffers, double buffered: index = buf * B + b
  double* cart_err;            // [2][B][n_cart_rows]
  double* cart_jac;            // [2][B][n_cart_rows][cart_stride]
  double* coll_rows;           // [2][B][n_coll_cand][coll_stride]
  unsigned long long* coll_mask;  // [2][B][n_coll_objs * coll_words]
  int n_coll_objs, pad2;
  // QP workspace (per trajectory)
  double* rows;                // [B][max_rows][row_stride]
  int* row_ints;               // [B][max_rows][RI_NINTS]
  int* lists;                  // [B][list_stride]: column pointers, column entries, object row ranges
  size_t list_stride;
  double* ws_x;                // [B][N]  warm start: previous QP solution (trajectory part, unscaled)
  double* ws_yb;               // [B][N]  warm start: duals of the variable-bound rows (unscaled)
  double* scratch;             // [B][5*Np]: dx dy stash(x zb yb)
  double* soa;                 // [grid][soa_stride]: column-major copy of a QP's rows while an ADMM block runs on rows that do
  size_t soa_stride;           //                     not fit shared memory (qp_soa_doubles)
  double* factor_g;            // [grid][3*M*nb*nb]: per-CTA home of a block-cyclic-reduction factor that does not fit
                               // shared memory (14 joints: blocks of 28); stays L2 resident
  int* lvs_overflow;           // [B] 1: a step pair had more active continuous-collision contacts than its row block holds
  int* qp_done;                // [B] 1: a QP solution is waiting for its evaluation
  int* ws_meta;                // [B][8]: warm-start key (n_aux, rows, nnzA, last status)
  double* ws_rho;              // [B]
  double* trace;               // [B][trace_cap][14] decision trace (same columns as the oracle's TraceEntry)
  int* trace_len;              // [B]
  int trace_cap, pad3;
  int* qp_paths;               // [B] QpPath bits of every QP since the start of the solve (nullptr: not recorded)
  double* dbg;                 // [B][16] solver diagnostics of the last QP (residuals, polish residuals, rho, c)
  int* sched_state;            // [B] persistent SQP kernel: 0 ready, 1 running, 2 finished
  unsigned long long* sched_timers;  // [4] ns in QP steps, ns in evaluation steps, evaluation steps, claims
  unsigned long long* clock_start;   // [1] %globaltimer ns at the start of the solve: the clock of every max_time
  int* sqp_top;                // [B] 1: the next QP of the trajectory begins a new SQP iteration (the time-limit check)
  int* ended_by;               // [B] what ended the trajectory: 0 its own SQP, 1 its max_time, 2 its group (group_stop)
  int* group_done;             // [B / group_size] 1: a seed of the group ended OPT_CONVERGED by its own SQP (group_stop)
  int group_size;              // seeds per problem: trajectories [g*G, (g+1)*G) are group g; 1 without groups
  int group_stop;              // 1: the siblings of a converged seed end at their next SQP iteration top (only with G > 1)
  QpSettings qp;
  int qp_fast_passes;  // 1: short trajectories take the fused termination check and polish_passes (qp_cta_kernel.cuh)
};

// Record layout of the SQP iteration log: a header of kLogHeader doubles, then n_cnts merit coefficients, the model values
// (n_costs, n_cnts), the exact values at the record's point (n_costs, n_cnts) and, with log_with_x, the point [T][D].
enum LogField {
  LOG_KIND = 0, LOG_ROUND, LOG_ITER, LOG_TRUST, LOG_OLD_MERIT, LOG_MODEL_MERIT, LOG_NEW_MERIT, LOG_QP_STATUS,
  LOG_ADMM_ITERS, LOG_ACTION, LOG_PRI_RES, LOG_DUA_RES, LOG_RHO, LOG_POLISH, LOG_WARM, LOG_ENDED, kLogHeader
};

}  // namespace tb200
