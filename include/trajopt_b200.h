/*
 * trajopt_b200.h — C ABI of the H100-native (sm_90a) batched SQP trajectory optimizer.
 *
 * This header is the drop-in boundary for ONE path of tesseract-robotics/trajopt:
 * sco::BasicTrustRegionSQP::optimize() (trajopt_sco/src/optimizers.cpp:699-991) with its
 * convexify step (trajopt/src/{trajectory_costs,kinematic_terms,collision_terms}.cpp) and
 * its QP subproblem solve (trajopt_sco/src/osqp_interface.cpp:440-615 -> OSQP), batched
 * over B independent trajectories.  The reference has no C ABI for this path (its ABI is
 * C++ virtuals: sco::Model, sco::Cost, sco::Constraint); the POD structs below are the
 * flattened form of what trajopt::ConstructProblem() produces from a
 * trajopt::ProblemConstructionInfo (trajopt/include/trajopt/problem_description.hpp:235-259).
 * The C++ host layer include/trajopt_b200.hpp re-exposes it under the reference's own names
 * (ProblemConstructionInfo / TermInfo subclasses / ModelType / BasicTrustRegionSQPParameters /
 * ConstructProblem / OptResults).
 *
 * Conventions: plain pointers + sizes, caller-owned buffers, int return codes
 * (0 = ok), no exceptions cross the boundary, thread-local tb200_last_error().
 * All real arithmetic is IEEE fp64 (sco::DblVec = std::vector<double>,
 * trajopt_sco/include/trajopt_sco/sco_common.hpp:17).
 */
#ifndef TRAJOPT_B200_H
#define TRAJOPT_B200_H

#include <math.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB200_VERSION_MAJOR 0
#define TB200_VERSION_MINOR 5
#define TB200_MAX_DOF 16      /* joints per manipulator group (7 single arm, 14 dual arm) */
#define TB200_MAX_STEPS 64    /* waypoints per trajectory */
#define TB200_MIN_CAST_ROWS_PER_PAIR 128  /* continuous collision evaluators: lower / upper limit of the active contacts */
#define TB200_MAX_CAST_ROWS_PER_PAIR 4096 /* (rows) one step pair can hold; see tb200inl_cast_rows_per_pair */

/* ---- return codes ------------------------------------------------------- */
enum {
  TB200_OK = 0,
  TB200_ERR_INVALID = 1,     /* bad argument / inconsistent description (PRINT_AND_THROW in the reference) */
  TB200_ERR_UNSUPPORTED = 2, /* term or option outside the implemented hot path */
  TB200_ERR_CUDA = 3,        /* CUDA runtime failure; the library never falls back to the CPU */
  TB200_ERR_NO_DEVICE = 4
};

/* sco::OptStatus, trajopt_sco/include/trajopt_sco/optimizers.hpp:25-33 (same numeric values) */
enum {
  TB200_OPT_CONVERGED = 0,
  TB200_OPT_SCO_ITERATION_LIMIT = 1,
  TB200_OPT_PENALTY_ITERATION_LIMIT = 2,
  TB200_OPT_TIME_LIMIT = 3,
  TB200_OPT_FAILED = 4,
  TB200_OPT_INVALID = 5
};

/* sco::CvxOptStatus, trajopt_sco/include/trajopt_sco/solver_interface.hpp:46-51 */
enum { TB200_CVX_SOLVED = 0, TB200_CVX_INFEASIBLE = 1, TB200_CVX_FAILED = 2 };

/* ---- robot -------------------------------------------------------------- */
enum { TB200_JOINT_FIXED = 0, TB200_JOINT_REVOLUTE = 1, TB200_JOINT_PRISMATIC = 2 };

/* One URDF joint+child link.  Frame i = parent frame * origin * motion(q).  Segments are
 * topologically ordered (parent index < own index); parent -1 = scene root.  This is the
 * data tesseract::kinematics::JointGroup::calcFwdKin consumes (called from
 * trajopt/src/kinematic_terms.cpp:252, collision_terms.cpp:415). */
typedef struct tb200_segment {
  int32_t parent;
  int32_t joint_type;
  int32_t q_index;          /* column of the trajectory this joint reads, -1 when fixed */
  int32_t reserved;
  double origin_xyz[3];
  double origin_wxyz[4];    /* unit quaternion of the joint origin rotation */
  double axis[3];           /* unit axis in the joint frame */
} tb200_segment;

/* Collision sphere rigidly attached to a segment frame (synthetic robot collision model,
 * SURVEY.md §8d: the reference uses Bullet convex meshes, which are unpinned). */
typedef struct tb200_sphere {
  int32_t segment;
  int32_t reserved;
  double center[3];         /* in the segment frame */
  double radius;
} tb200_sphere;

typedef struct tb200_robot {
  int32_t n_dof;
  int32_t n_segments;
  const tb200_segment* segments;
  const double* lower;      /* [n_dof] joint limits (kin->getLimits(), problem_description.cpp:556-559) */
  const double* upper;
  int32_t n_spheres;
  int32_t reserved;
  const tb200_sphere* spheres;
} tb200_robot;

/* ---- terms (trajopt::TermInfo subclasses, problem_description.hpp:273-659) ------------ */
enum {
  TB200_TERM_JOINT_POS = 0,  /* JointPosTermInfo  -> trajectory_costs.cpp:12-254   */
  TB200_TERM_JOINT_VEL = 1,  /* JointVelTermInfo  -> trajectory_costs.cpp:257-499  */
  TB200_TERM_JOINT_ACC = 2,  /* JointAccTermInfo  -> trajectory_costs.cpp:502-754  */
  TB200_TERM_CART_POSE = 3,  /* CartPoseTermInfo  -> kinematic_terms.cpp:187-366   */
  TB200_TERM_CART_VEL = 4,   /* CartVelTermInfo   -> kinematic_terms.cpp:368-425   */
  TB200_TERM_COLLISION = 5,  /* CollisionTermInfo -> collision_terms.cpp            */
  TB200_TERM_AVOID_SINGULARITY = 6 /* AvoidSingularityTermInfo -> kinematic_terms.cpp:586-642 */
};
enum { TB200_ROLE_COST = 1, TB200_ROLE_CNT = 2 }; /* TermType::TT_COST / TT_CNT */

/* tesseract CollisionEvaluatorType as read by CollisionTermInfo::fromJson
 * (problem_description.cpp:1617-1712): 1 DISCRETE, 2 LVS_DISCRETE, 3 CONTINUOUS, 4 LVS_CONTINUOUS */
enum { TB200_COLL_DISCRETE = 1, TB200_COLL_LVS_DISCRETE = 2, TB200_COLL_CONTINUOUS = 3, TB200_COLL_LVS_CONTINUOUS = 4 };

typedef struct tb200_term {
  int32_t kind;
  int32_t role;
  int32_t first_step;       /* inclusive; CART_POSE: the timestep */
  int32_t last_step;        /* inclusive (already clamped the way TermInfo::hatch does) */
  /* joint terms: all-zero tolerances => Eq flavour, else Ineq flavour */
  double coeffs[TB200_MAX_DOF];
  double targets[TB200_MAX_DOF];
  double upper_tols[TB200_MAX_DOF];
  double lower_tols[TB200_MAX_DOF];
  /* cartesian terms */
  int32_t link;             /* segment whose frame is the moving (source) frame / CartVel link */
  int32_t target_slot;      /* >=0: read the static target pose from cart_targets[b][slot]; -1: use target_pose */
  double source_offset[7];  /* xyz + wxyz, applied on the right of the link frame */
  double target_pose[7];    /* target_frame * target_frame_offset expressed in the scene root */
  double pos_coeffs[3];
  double rot_coeffs[3];
  double max_displacement;  /* CartVel */
  /* collision */
  int32_t evaluator_type;
  int32_t n_fixed_steps;
  int32_t fixed_steps[8];
  double margin;            /* "dist_pen" */
  double coeff;
  double margin_buffer;     /* collision_margin_buffer: rows are emitted out to margin+buffer */
  double longest_valid_segment_length;
  /* AVOID_SINGULARITY: one object per step in [first_step, last_step] on the geometric Jacobian of `link` (all
   * n_dof columns); error 1/(s + lambda) - 1/(0.1 + lambda) with s the smallest singular value, scaled by coeffs[0]
   * (1: unscaled).  COST: ABS penalty (also penalises s above 0.1); CNT: INEQ constraint (s >= 0.1).  One row of
   * the Cartesian row buffers per object.  lambda is the damping of the term (the reference's default is 0.1; a
   * zeroed struct holds 0, so callers set it); it must be finite and >= 0. */
  double lambda;
} tb200_term;

/* sco::BasicTrustRegionSQPParameters, optimizers.hpp:92-135 (same defaults via tb200_default_sqp_params) */
typedef struct tb200_sqp_params {
  double improve_ratio_threshold;
  double min_trust_box_size;
  double min_approx_improve;
  double min_approx_improve_frac;
  int32_t max_iter;
  int32_t max_qp_solver_failures;
  double trust_shrink_ratio;
  double trust_expand_ratio;
  double cnt_tolerance;
  double max_merit_coeff_increases;
  double merit_coeff_increase_ratio;
  double initial_merit_error_coeff;
  double trust_box_size;
  int32_t inflate_constraints_individually;
  int32_t reserved;
  /* wall-clock budget of a solve in seconds (optimizers.cpp:738-753); DBL_MAX = none.  Checked at the top of every SQP
   * iteration: a trajectory past it ends with its last accepted iterate, OPT_CONVERGED when its constraints are within
   * cnt_tolerance (or it has none), else OPT_TIME_LIMIT.  One device clock per solve (DESIGN.md section 6). */
  double max_time;
} tb200_sqp_params;

/* OSQPSettings as set by OSQPModelConfig::setDefaultOSQPSettings (osqp_interface.cpp:78-90)
 * on top of osqp_set_default_settings (OSQP v1.0.0, not in the reference tree). */
typedef struct tb200_qp_settings {
  double rho;               /* 0.1 */
  double sigma;             /* 1e-6 */
  double alpha;             /* 1.6 */
  double eps_abs;           /* 1e-4 (reference) */
  double eps_rel;           /* 1e-6 (reference) */
  double eps_prim_inf;      /* 1e-4 */
  double eps_dual_inf;      /* 1e-4 */
  double delta;             /* 1e-6 polish regularisation */
  double adaptive_rho_tolerance; /* 5 */
  int32_t max_iter;         /* 8192 (reference) */
  int32_t scaling;          /* 10 Ruiz passes */
  int32_t check_termination;/* 25 */
  int32_t adaptive_rho;     /* 1 (reference) */
  int32_t adaptive_rho_interval; /* 50: fixed (OSQP's default is wall-clock based => not reproducible) */
  int32_t polishing;        /* 1 (reference) */
  int32_t polish_refine_iter; /* 3 */
  int32_t warm_starting;    /* 1 */
  int32_t early_polish_every; /* 25: also try the VERIFIED polish at every such check before ADMM has met its own
                                 tolerances (DESIGN.md optimisation O1; same QP minimiser, fewer iterations);
                                 0 = OSQP's order (polish only after ADMM converged) */
  int32_t early_polish_from;  /* 25: first iteration at which the early polish is tried */
} tb200_qp_settings;

typedef struct tb200_problem_desc {
  tb200_robot robot;
  int32_t n_steps;          /* T  (basic_info.n_steps) */
  int32_t batch;            /* B independent trajectories sharing this description */
  int32_t n_terms;
  int32_t n_fixed_timesteps;/* basic_info.fixed_timesteps */
  const tb200_term* terms;  /* cost_infos first, then cnt_infos, in pci order */
  const int32_t* fixed_timesteps;
  int32_t n_fixed_dofs;     /* basic_info.fixed_dofs */
  int32_t n_cart_targets;   /* per-trajectory target slots */
  const int32_t* fixed_dofs;
  const double* init_traj;  /* [B][T][D] row-major = trajToDblVec(prob->GetInitTraj()) per trajectory */
  const double* cart_targets; /* [B][n_cart_targets][7] xyz+wxyz, may be NULL */
  int32_t n_obstacles;      /* static world spheres */
  int32_t obstacles_per_traj; /* 1: obstacles is [B][O][4]; 0: [O][4] shared */
  const double* obstacles;  /* (x,y,z,r) in the scene root frame */
  tb200_sqp_params sqp;
  tb200_qp_settings qp;
  /* Multi-start solves (not in the reference; DESIGN.md section 4.1).  group_size G >= 2: trajectories [g*G, (g+1)*G) are
   * G seeds of problem g (batch % G == 0); 0 or 1: no groups.  group_stop 1: a seed that ends OPT_CONVERGED by its own
   * SQP ends its running siblings at their next SQP iteration top, under the time-limit rule (last accepted iterate;
   * OPT_CONVERGED when its constraints are within cnt_tolerance, else OPT_TIME_LIMIT); 0: every seed runs to its end.
   * The best seed of every group is selected on the device (tb200_fetch_group_results). */
  int32_t group_size;
  int32_t group_stop;
  /* Per-trajectory optimizer parameters (not in the reference; DESIGN.md section 4.1): [batch] rows, trajectory b runs
   * under row b (every field, max_time against the one clock of the batch); NULL: `sqp` for every trajectory. */
  const tb200_sqp_params* sqp_per_traj;
} tb200_problem_desc;

/* Caller-owned result buffers = sco::OptResults per trajectory (optimizers.hpp:40-59).
 * Any pointer may be NULL to skip that output. */
typedef struct tb200_results {
  double* x;                /* [B][T][D] */
  int32_t* status;          /* [B] TB200_OPT_* */
  double* total_cost;       /* [B] */
  double* cost_vals;        /* [B][n_costs] */
  double* cnt_viols;        /* [B][n_cnts]  (EQ objects first, then INEQ — modeling.cpp:234-241) */
  int32_t* n_qp_solves;     /* [B] */
  int32_t* n_func_evals;    /* [B] */
  int32_t* n_admm_iters;    /* [B] total ADMM iterations spent (diagnostic, not in the reference) */
} tb200_results;

/* Fixed-layout output of one batched convexify pass (kernel-level parity tests).
 * Row r of trajectory b linearises one scalar error:  value(q) ~ constant + coeffs.(q - q0)
 * around the waypoint(s) it reads. */
typedef struct tb200_convexify_out {
  double* cart_err;         /* [B][n_cart_rows]          coeff-scaled CartPose/CartVel/AvoidSingularity errors at x */
  double* cart_jac;         /* [B][n_cart_rows][cart_jac_stride] coeff-scaled Jacobian rows                     */
  double* coll_rows;        /* [B][n_coll_cand][coll_row_stride]: grad[0..nvar-1], dist0, margin, coeff, active */
  double* cost_vals;        /* [B][n_costs]  exact Cost::value(x)           */
  double* cnt_viols;        /* [B][n_cnts]   exact Constraint::violation(x) */
} tb200_convexify_out;

typedef struct tb200_layout {
  int32_t n_costs;          /* sco::Cost objects hatched       */
  int32_t n_cnts;           /* sco::Constraint objects hatched */
  int32_t n_cart_rows;
  int32_t cart_jac_stride;
  int32_t n_coll_cand;      /* dense candidate collision rows per trajectory */
  int32_t coll_row_stride;
  int32_t n_vars;           /* T*D */
  int32_t reserved;
} tb200_layout;

/* Rows (active contacts) one step pair of a continuous collision term can hold.  The LVS sub-trajectory itself is as
 * long as the reference's (ceil(dist / lvs) sub-segments, collision_terms.cpp:1118-1155, unbounded) and only contacts
 * inside margin + buffer take a row, but the row block of a pair has a fixed size: room for EVERY candidate (robot
 * sphere x obstacle x sub-segment) of the longest step pair of the description's initial trajectories, rounded up to 64,
 * within [TB200_MIN_CAST_ROWS_PER_PAIR, TB200_MAX_CAST_ROWS_PER_PAIR].  (The reference's JSON default of
 * collision_margin_buffer is 0.5 m: nearly every candidate near an obstacle is an active contact then.)  A step pair that
 * comes to hold more during a solve is never truncated: its trajectory ends OPT_FAILED and the solve returns
 * TB200_ERR_UNSUPPORTED.  The CPU oracle sizes its row output with the same function. */
static inline int tb200inl_cast_rows_per_pair(const tb200_problem_desc* d) {
  const int T = d->n_steps, D = d->robot.n_dof;
  double need = 1.0;
  for (int k = 0; k < d->n_terms; ++k) {
    const tb200_term* tm = d->terms + k;
    if (tm->kind != TB200_TERM_COLLISION) continue;
    if (tm->evaluator_type == TB200_COLL_LVS_DISCRETE && need < 2.0) need = 2.0; /* both waypoints are tested */
    if (tm->evaluator_type != TB200_COLL_LVS_CONTINUOUS && tm->evaluator_type != TB200_COLL_LVS_DISCRETE) continue;
    if (!(tm->longest_valid_segment_length > 0.0)) continue;
    for (int b = 0; b < d->batch; ++b)
      for (int t = tm->first_step < 0 ? 0 : tm->first_step; t < tm->last_step && t + 1 < T; ++t) {
        const double* q0 = d->init_traj + ((size_t)b * T + t) * D;
        double s = 0.0;
        for (int j = 0; j < D; ++j) s += (q0[D + j] - q0[j]) * (q0[D + j] - q0[j]);
        s = sqrt(s);
        if (s > tm->longest_valid_segment_length) {
          /* sub-segments (continuous) | states (LVS_DISCRETE: one more) of this step pair */
          const double n = ceil(s / tm->longest_valid_segment_length) + (tm->evaluator_type == TB200_COLL_LVS_DISCRETE ? 1.0 : 0.0);
          if (n > need) need = n;
        }
      }
  }
  {
    double cand = need * (double)d->robot.n_spheres * (double)d->n_obstacles;
    cand = ceil(cand / 64.0) * 64.0;
    if (cand < TB200_MIN_CAST_ROWS_PER_PAIR) cand = TB200_MIN_CAST_ROWS_PER_PAIR;
    if (cand > TB200_MAX_CAST_ROWS_PER_PAIR) cand = TB200_MAX_CAST_ROWS_PER_PAIR;
    return (int)cand;
  }
}

typedef struct tb200_problem tb200_problem; /* opaque handle; not thread-safe */

const char* tb200_version(void);
const char* tb200_last_error(void);
void tb200_default_sqp_params(tb200_sqp_params* p);
void tb200_default_qp_settings(tb200_qp_settings* s);

/* Validates + uploads the description (deep copy; caller may free its arrays afterwards).
 * device: CUDA ordinal.  Replaces trajopt::ConstructProblem's sco::OptProb assembly
 * (problem_description.cpp:410-542) for the batched path. */
int tb200_problem_create(const tb200_problem_desc* desc, int device, tb200_problem** out);
void tb200_problem_destroy(tb200_problem* p);
int tb200_problem_layout(const tb200_problem* p, tb200_layout* out);

/* Replace the optimizer parameters of an existing problem (what `opt.getParameters() = ...` does on a
 * sco::BasicTrustRegionSQP, optimizers.hpp:92-135, 365-366), for every trajectory: a per-trajectory table is dropped.
 * Takes effect at the next solve. */
int tb200_problem_set_sqp_params(tb200_problem* p, const tb200_sqp_params* params);
/* Per-trajectory optimizer parameters: rows [batch], trajectory b runs under rows[b] (as tb200_problem_desc.sqp_per_traj);
 * NULL drops the table, and every trajectory runs under the uniform parameters again.  Takes effect at the next solve. */
int tb200_problem_set_sqp_params_per_traj(tb200_problem* p, const tb200_sqp_params* rows);

/* Replace the per-trajectory inputs without rebuilding (same shapes). Host pointers. */
int tb200_problem_set_inputs(tb200_problem* p, const double* init_traj, const double* cart_targets,
                             const double* obstacles);

/* Whole hot path: BasicTrustRegionSQP::optimize() for all B trajectories
 * (optimizers.cpp:699-991).  HOST buffers in and out; H2D/D2H inside the call. */
int tb200_solve_batch(tb200_problem* p, tb200_results* out);

/* Same, inputs already resident on the device (set_inputs was called); results stay on the
 * device until tb200_fetch_results.  Used for the HBM-resident bench leg. */
int tb200_solve_batch_resident(tb200_problem* p);
int tb200_fetch_results(tb200_problem* p, tb200_results* out);

/* Replace group_size / group_stop of an existing problem (same rules as in tb200_problem_desc).  Takes effect at the
 * next solve. */
int tb200_problem_set_groups(tb200_problem* p, int32_t group_size, int32_t group_stop);

/* Per-group results of the last solve; NG = batch / group_size groups (without groups every trajectory is its own
 * group, NG = batch).  The best seed of a group is the minimum of the key
 *   (status != OPT_CONVERGED, status != OPT_CONVERGED ? max(cnt_viols) : 0, total_cost, batch index)
 * with a NaN read as +inf.  Any pointer may be NULL to skip that output. */
typedef struct tb200_group_results {
  int32_t* best;            /* [NG] batch index of the best seed */
  int32_t* status;          /* [NG] its status */
  double* total_cost;       /* [NG] its total cost */
  double* x;                /* [NG][T][D] its trajectory */
  int32_t* n_converged;     /* [NG] seeds of the group that ended OPT_CONVERGED */
  int32_t* ended_by;        /* [batch] per trajectory: 0 its own SQP, 1 the time limit (max_time), 2 its group */
} tb200_group_results;
int tb200_fetch_group_results(tb200_problem* p, tb200_group_results* out);

/* Kernel-level entry points for parity tests.
 * x: host [B][T][D].  Equivalent of costs[i]->convex/value + cnts[i]->convex/violation
 * (optimizers.cpp:761-783) at x for every trajectory. */
int tb200_convexify_batch(tb200_problem* p, const double* x, tb200_convexify_out* out);

/* One Model::optimize() per trajectory (optimizers.cpp:813-814) on the QP convexified at x
 * with trust box size trust[b] and penalty coefficients merit_coeffs[b][n_cnts].
 * Outputs: new_x [B][T][D], qp_status [B] TB200_CVX_*, model_cost_vals [B][n_costs],
 * model_cnt_viols [B][n_cnts], admm_iters [B]. */
int tb200_qp_solve_batch(tb200_problem* p, const double* x, const double* trust, const double* merit_coeffs,
                         double* new_x, int32_t* qp_status, double* model_cost_vals, double* model_cnt_viols,
                         int32_t* admm_iters);

/* ---- general QP (the sco::Model plugin surface, include/trajopt_b200_sco.hpp) ----------------------------
 * OSQP's canonical form as OSQPModel builds it (trajopt_sco/src/osqp_interface.cpp:170-281):
 *     min 1/2 x'Px + q'x   s.t.  l <= A x <= u        (variable bounds are identity rows of A)
 * with dense, row-major inputs; `batch` problems of the same size back to back.  Replaces
 * OSQPModel::optimize() -> osqp_setup / osqp_solve (osqp_interface.cpp:283-370, 440-615) for one
 * sco::Model::optimize() call at a time; the batched trajectory path does not go through it. */
typedef struct tb200_qp_general {
  int32_t n;                /* variables */
  int32_t m;                /* rows of A */
  int32_t batch;            /* problems (>= 1) */
  int32_t reserved;
  const double* P;          /* [batch][n][n] symmetric; the upper triangle is read */
  const double* q;          /* [batch][n] */
  const double* A;          /* [batch][m][n] */
  const double* l;          /* [batch][m]  (<= -1e30: none) */
  const double* u;          /* [batch][m]  (>=  1e30: none) */
} tb200_qp_general;
/* OSQP status values (osqp_api_constants.h): 1 solved, 2 solved inaccurate, 3/4 primal infeasible (/inaccurate),
 * 5/6 dual infeasible (/inaccurate), 7 max iterations, 8 non convex */
int tb200_qp_solve_general(const tb200_qp_general* qp, const tb200_qp_settings* settings /* NULL: defaults */, int device,
                           double* x /* [batch][n] */, double* y /* [batch][m] or NULL */, int32_t* status /* [batch] */,
                           int32_t* iters /* [batch] or NULL */, int32_t* polish /* [batch] or NULL */);
const char* tb200_qp_general_last_error(void);

/* OSQP's own order of operations: the polish runs only after ADMM has met its tolerances
 * (tb200_default_qp_settings also tries the VERIFIED polish early, DESIGN.md optimisation O1). */
void tb200_osqp_order_qp_settings(tb200_qp_settings* s);

/* Polish outcome (1 accepted, -1 rejected, 0 not attempted) of the last tb200_qp_solve_batch call, [B]. */
int tb200_last_qp_polish(tb200_problem* p, int32_t* polish);

/* ---- trajectory collision check (tesseract's checkTrajectory; DESIGN.md section 4.6) ----------------------------
 * Every trajectory of the batch against the problem's robot spheres and its current obstacles (as last set by
 * tb200_problem_create or tb200_problem_set_inputs).  Every waypoint or step pair is checked: fixed steps and the
 * margin buffer of the collision terms play no part.  A contact is a (robot sphere, obstacle) pair with signed distance
 * < margin (0: penetration).  type is one of TB200_COLL_*, with the sub-trajectory rules of the collision terms:
 *   DISCRETE        S = T slots, one per waypoint; sphere/sphere distance.
 *   LVS_DISCRETE    S = T-1 slots, one per step pair; the states q0 + (q1-q0) i/n, i = 0..n, n = ceil(|q1-q0| / lvs)
 *                   (1 when the step is no longer than lvs), both waypoints included.
 *   CONTINUOUS      S = T-1; one swept test per pair: the capsule of each sphere centre's path between the two states
 *                   (the chord of the true centre path) against the obstacle sphere.
 *   LVS_CONTINUOUS  S = T-1; n swept sub-segments per pair.
 * n has no cap.  Per slot: the minimum signed distance, the number of contacts counted over (sphere, obstacle,
 * sub-state | sub-segment) triples, and the argmin (sphere, obstacle, sub-index) with ties to the lowest index in that
 * order.  Spheres are numbered as in the description.  A non-finite distance counts as a contact and is reported as
 * NaN.  Without spheres or obstacles: +inf, no contacts, argmin (-1, -1, -1). */
typedef struct tb200_check_config {
  int32_t type;             /* TB200_COLL_* */
  int32_t reserved;
  double longest_valid_segment_length; /* LVS types: > 0 */
  double margin;            /* contact: distance < margin */
} tb200_check_config;
/* Caller-owned; any pointer may be NULL to skip that output.  S = T for DISCRETE, else T-1. */
typedef struct tb200_check_results {
  double* step_min_distance; /* [B][S] */
  int32_t* step_contacts;    /* [B][S] */
  int32_t* step_argmin;      /* [B][S][3] sphere, obstacle, sub-index */
  int32_t* in_collision;     /* [B] 1: some slot has a contact */
  int32_t* first_slot;       /* [B] first slot with a contact, -1 if none */
  double* min_distance;      /* [B] minimum over the slots (NaN if a slot's is) */
} tb200_check_results;
/* x: host [B][T][D], or NULL for the x of the last solve, already on the device (tb200_solve_batch_resident -> check ->
 * fetch needs no round trip).  TB200_ERR_INVALID for an unknown type, an LVS type with lvs <= 0 or NaN, a non-finite
 * margin, and a NULL x before any solve. */
int tb200_check_trajectories(tb200_problem* p, const double* x, const tb200_check_config* cfg, tb200_check_results* out);

/* ---- SQP iteration log (DESIGN.md section 4.7) --------------------------------------------------------------------
 * Opt-in record of what every trajectory's SQP did, written on the device by the decision step.  capacity R > 0: the
 * next solves keep up to R records per trajectory (later ones are counted in n_dropped and not written, so the records
 * kept are always the same prefix); with_x 1: each record also holds its point [T][D].  0: off (the default).  Takes
 * effect at the next solve; the log of a solve stays readable until the next one.  TB200_ERR_INVALID for a negative
 * capacity, a with_x other than 0 or 1, and a buffer (batch x R x record size) that cannot be addressed.  Solves with
 * and without the log compute the same results, bit for bit; tb200_convexify_batch and tb200_qp_solve_batch write no
 * records. */
int tb200_problem_set_sqp_log(tb200_problem* p, int32_t capacity, int32_t with_x);

/* The log of the last solve.  Per trajectory b, records r < n_records[b] in order: record 0 (kind 0) is the state after
 * the initial evaluation (the clamped start point, its exact values, the initial merit coefficients and trust box);
 * then one record (kind 1) per QP solve, failed ones included, in the order of n_qp_solves.  A trajectory ended by the
 * time limit or by its group simply has no more records.  Arrays are [B][R](...) with R = the capacity the solve ran
 * with; entries past n_records[b] are 0 / -1 / NaN.  Any pointer may be NULL to skip that output. */
typedef struct tb200_sqp_log {
  int32_t* n_records;       /* [B] records kept (n_qp_solves + 1 when nothing was dropped) */
  int32_t* n_dropped;       /* [B] records that did not fit */
  int32_t* kind;            /* [B][R] 0 initial state, 1 QP solve */
  int32_t* merit_round;     /* [B][R] merit coefficient round the QP belongs to (0-based) */
  int32_t* iter;            /* [B][R] SQP iteration within that round (1-based) */
  double* trust_box_size;   /* [B][R] trust box the QP was solved with (kind 0: the initial one) */
  int32_t* qp_status;       /* [B][R] QP solver status (OSQP's values, see tb200_qp_solve_general); -1 for kind 0 */
  int32_t* admm_iters;      /* [B][R] ADMM iterations of the QP */
  int32_t* polish;          /* [B][R] 1 polish accepted, -1 rejected, 0 not attempted */
  double* qp_diag;          /* [B][R][4] primal residual, dual residual, final rho, 1 if warm started */
  int32_t* action;          /* [B][R] 0 trust box shrunk, 1 step accepted, 2 converged by small improvement, 3 QP
                               failure; -1 for kind 0 */
  int32_t* ended;           /* [B][R] TB200_OPT_* the trajectory ended with at this record, -1: it went on */
  double* old_merit;        /* [B][R] merit at the last accepted point; NaN for kind 0 and a failed QP */
  double* model_merit;      /* [B][R] merit of the QP model at its solution; NaN likewise */
  double* new_merit;        /* [B][R] exact merit at the QP solution; NaN likewise */
  double* merit_coeffs;     /* [B][R][n_cnts] merit coefficients the decision used */
  double* model_cost_vals;  /* [B][R][n_costs] model value of every cost at the QP solution, as summed into model_merit */
  double* model_cnt_viols;  /* [B][R][n_cnts] NaN for kind 0 and a failed QP */
  double* old_cost_vals;    /* [B][R][n_costs] exact values at the last accepted point (filled on the host) */
  double* old_cnt_viols;    /* [B][R][n_cnts]  NaN for kind 0 */
  double* new_cost_vals;    /* [B][R][n_costs] exact values at the record's point (kind 0: the start; NaN: failed QP) */
  double* new_cnt_viols;    /* [B][R][n_cnts] */
  double* new_x;            /* [B][R][T][D] the record's point; only when the log was recorded with_x */
} tb200_sqp_log;
int tb200_fetch_sqp_log(tb200_problem* p, tb200_sqp_log* out);

/* The sco::Cost / sco::Constraint objects of the problem in OptProb order (costs, then equality constraints, then
 * inequality constraints: the order of cost_vals and cnt_viols): term[i] = index in desc.terms of the term that hatched
 * object i, step[i] = its step (joint terms: their first step; collision and CartVel: the step or first step of the
 * pair).  n_costs + n_cnts entries each (tb200_problem_layout); either pointer may be NULL. */
int tb200_problem_objects(const tb200_problem* p, int32_t* term, int32_t* step);

/* Timing of the last tb200_solve_batch* call, measured with CUDA events on the solver's
 * stream: total ms, convexify-kernel ms and launches, qp-kernel ms and launches. */
typedef struct tb200_timing {
  double total_ms;
  double convexify_ms;
  double qp_ms;
  double merit_ms;
  int32_t convexify_launches;
  int32_t qp_launches;
  int32_t merit_launches;
  int32_t outer_steps;
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int64_t convexify_bytes; /* algorithmic HBM bytes moved by all convexify launches */
} tb200_timing;
int tb200_last_timing(const tb200_problem* p, tb200_timing* out);

#ifdef __cplusplus
}
#endif
#endif /* TRAJOPT_B200_H */
