"""ctypes mirror of include/trajopt_b200.h (the C-ABI drop-in boundary).

The structs here are byte-for-byte the PODs of the header; `ProblemDesc` owns the numpy
buffers the C side points into.  `load_library()` loads the in-tree CUDA build
(trajopt_b200/csrc/libtrajopt_b200.so) and raises if it is missing: there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

MAX_DOF = 16

# enums (include/trajopt_b200.h)
JOINT_FIXED, JOINT_REVOLUTE, JOINT_PRISMATIC = 0, 1, 2
# return codes of the C ABI (include/trajopt_b200.h)
OK, ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_NO_DEVICE = range(5)
TERM_JOINT_POS, TERM_JOINT_VEL, TERM_JOINT_ACC, TERM_CART_POSE, TERM_CART_VEL, TERM_COLLISION, TERM_AVOID_SINGULARITY = range(7)
ROLE_COST, ROLE_CNT = 1, 2
COLL_DISCRETE, COLL_LVS_DISCRETE, COLL_CONTINUOUS, COLL_LVS_CONTINUOUS = 1, 2, 3, 4
OPT_CONVERGED, OPT_SCO_ITERATION_LIMIT, OPT_PENALTY_ITERATION_LIMIT, OPT_TIME_LIMIT, OPT_FAILED, OPT_INVALID = range(6)
CVX_SOLVED, CVX_INFEASIBLE, CVX_FAILED = range(3)

_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


class Segment(C.Structure):
    _fields_ = [("parent", C.c_int32), ("joint_type", C.c_int32), ("q_index", C.c_int32), ("reserved", C.c_int32),
                ("origin_xyz", C.c_double * 3), ("origin_wxyz", C.c_double * 4), ("axis", C.c_double * 3)]


class Sphere(C.Structure):
    _fields_ = [("segment", C.c_int32), ("reserved", C.c_int32), ("center", C.c_double * 3), ("radius", C.c_double)]


class Robot(C.Structure):
    _fields_ = [("n_dof", C.c_int32), ("n_segments", C.c_int32), ("segments", C.POINTER(Segment)),
                ("lower", _dbl_p), ("upper", _dbl_p), ("n_spheres", C.c_int32), ("reserved", C.c_int32),
                ("spheres", C.POINTER(Sphere))]


class Term(C.Structure):
    _fields_ = [("kind", C.c_int32), ("role", C.c_int32), ("first_step", C.c_int32), ("last_step", C.c_int32),
                ("coeffs", C.c_double * MAX_DOF), ("targets", C.c_double * MAX_DOF),
                ("upper_tols", C.c_double * MAX_DOF), ("lower_tols", C.c_double * MAX_DOF),
                ("link", C.c_int32), ("target_slot", C.c_int32),
                ("source_offset", C.c_double * 7), ("target_pose", C.c_double * 7),
                ("pos_coeffs", C.c_double * 3), ("rot_coeffs", C.c_double * 3), ("max_displacement", C.c_double),
                ("evaluator_type", C.c_int32), ("n_fixed_steps", C.c_int32), ("fixed_steps", C.c_int32 * 8),
                ("margin", C.c_double), ("coeff", C.c_double), ("margin_buffer", C.c_double),
                ("longest_valid_segment_length", C.c_double),
                ("lambda_", C.c_double)]  # AvoidSingularity damping ("lambda" in the C header)


class SqpParams(C.Structure):
    _fields_ = [("improve_ratio_threshold", C.c_double), ("min_trust_box_size", C.c_double),
                ("min_approx_improve", C.c_double), ("min_approx_improve_frac", C.c_double),
                ("max_iter", C.c_int32), ("max_qp_solver_failures", C.c_int32),
                ("trust_shrink_ratio", C.c_double), ("trust_expand_ratio", C.c_double),
                ("cnt_tolerance", C.c_double), ("max_merit_coeff_increases", C.c_double),
                ("merit_coeff_increase_ratio", C.c_double), ("initial_merit_error_coeff", C.c_double),
                ("trust_box_size", C.c_double), ("inflate_constraints_individually", C.c_int32),
                ("reserved", C.c_int32), ("max_time", C.c_double)]


class QpSettings(C.Structure):
    _fields_ = [("rho", C.c_double), ("sigma", C.c_double), ("alpha", C.c_double), ("eps_abs", C.c_double),
                ("eps_rel", C.c_double), ("eps_prim_inf", C.c_double), ("eps_dual_inf", C.c_double),
                ("delta", C.c_double), ("adaptive_rho_tolerance", C.c_double), ("max_iter", C.c_int32),
                ("scaling", C.c_int32), ("check_termination", C.c_int32), ("adaptive_rho", C.c_int32),
                ("adaptive_rho_interval", C.c_int32), ("polishing", C.c_int32), ("polish_refine_iter", C.c_int32),
                ("warm_starting", C.c_int32), ("early_polish_every", C.c_int32), ("early_polish_from", C.c_int32)]


class ProblemDescC(C.Structure):
    _fields_ = [("robot", Robot), ("n_steps", C.c_int32), ("batch", C.c_int32), ("n_terms", C.c_int32),
                ("n_fixed_timesteps", C.c_int32), ("terms", C.POINTER(Term)), ("fixed_timesteps", _i32_p),
                ("n_fixed_dofs", C.c_int32), ("n_cart_targets", C.c_int32), ("fixed_dofs", _i32_p),
                ("init_traj", _dbl_p), ("cart_targets", _dbl_p), ("n_obstacles", C.c_int32),
                ("obstacles_per_traj", C.c_int32), ("obstacles", _dbl_p), ("sqp", SqpParams), ("qp", QpSettings),
                ("group_size", C.c_int32), ("group_stop", C.c_int32), ("sqp_per_traj", C.POINTER(SqpParams))]


class QpGeneral(C.Structure):
    """tb200_qp_general: dense QP(s) in OSQP's canonical form (include/trajopt_b200.h)."""
    _fields_ = [("n", C.c_int32), ("m", C.c_int32), ("batch", C.c_int32), ("reserved", C.c_int32), ("P", _dbl_p),
                ("q", _dbl_p), ("A", _dbl_p), ("l", _dbl_p), ("u", _dbl_p)]


class Results(C.Structure):
    _fields_ = [("x", _dbl_p), ("status", _i32_p), ("total_cost", _dbl_p), ("cost_vals", _dbl_p),
                ("cnt_viols", _dbl_p), ("n_qp_solves", _i32_p), ("n_func_evals", _i32_p), ("n_admm_iters", _i32_p)]


class GroupResults(C.Structure):
    _fields_ = [("best", _i32_p), ("status", _i32_p), ("total_cost", _dbl_p), ("x", _dbl_p), ("n_converged", _i32_p),
                ("ended_by", _i32_p)]


class ConvexifyOut(C.Structure):
    _fields_ = [("cart_err", _dbl_p), ("cart_jac", _dbl_p), ("coll_rows", _dbl_p), ("cost_vals", _dbl_p),
                ("cnt_viols", _dbl_p)]


class Layout(C.Structure):
    _fields_ = [("n_costs", C.c_int32), ("n_cnts", C.c_int32), ("n_cart_rows", C.c_int32),
                ("cart_jac_stride", C.c_int32), ("n_coll_cand", C.c_int32), ("coll_row_stride", C.c_int32),
                ("n_vars", C.c_int32), ("reserved", C.c_int32)]


class CheckConfig(C.Structure):
    """tb200_check_config: the trajectory collision check (type COLL_*, lvs for the LVS types, contact margin)."""
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("longest_valid_segment_length", C.c_double),
                ("margin", C.c_double)]


class CheckResults(C.Structure):
    _fields_ = [("step_min_distance", _dbl_p), ("step_contacts", _i32_p), ("step_argmin", _i32_p),
                ("in_collision", _i32_p), ("first_slot", _i32_p), ("min_distance", _dbl_p)]


class SqpLog(C.Structure):
    """tb200_sqp_log: the SQP iteration log of the last solve ([B][R](...) arrays, NULL-skippable)."""
    _fields_ = [("n_records", _i32_p), ("n_dropped", _i32_p), ("kind", _i32_p), ("merit_round", _i32_p), ("iter", _i32_p),
                ("trust_box_size", _dbl_p), ("qp_status", _i32_p), ("admm_iters", _i32_p), ("polish", _i32_p),
                ("qp_diag", _dbl_p), ("action", _i32_p), ("ended", _i32_p), ("old_merit", _dbl_p), ("model_merit", _dbl_p),
                ("new_merit", _dbl_p), ("merit_coeffs", _dbl_p), ("model_cost_vals", _dbl_p), ("model_cnt_viols", _dbl_p),
                ("old_cost_vals", _dbl_p), ("old_cnt_viols", _dbl_p), ("new_cost_vals", _dbl_p), ("new_cnt_viols", _dbl_p),
                ("new_x", _dbl_p)]


class Timing(C.Structure):
    _fields_ = [("total_ms", C.c_double), ("convexify_ms", C.c_double), ("qp_ms", C.c_double),
                ("merit_ms", C.c_double), ("convexify_launches", C.c_int32), ("qp_launches", C.c_int32),
                ("merit_launches", C.c_int32), ("outer_steps", C.c_int32), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("convexify_bytes", C.c_int64)]


def default_sqp_params():
    """sco::BasicTrustRegionSQPParameters defaults (trajopt_sco/include/trajopt_sco/optimizers.hpp:92-135)."""
    p = SqpParams()
    p.improve_ratio_threshold = 0.25
    p.min_trust_box_size = 1e-4
    p.min_approx_improve = 1e-4
    p.min_approx_improve_frac = -np.finfo(np.float64).max
    p.max_iter = 50
    p.max_qp_solver_failures = 3
    p.trust_shrink_ratio = 0.1
    p.trust_expand_ratio = 1.5
    p.cnt_tolerance = 1e-4
    p.max_merit_coeff_increases = 5
    p.merit_coeff_increase_ratio = 10
    p.initial_merit_error_coeff = 10
    p.trust_box_size = 0.1
    p.inflate_constraints_individually = 1
    p.max_time = np.finfo(np.float64).max  # seconds; no time limit
    return p


def default_qp_settings():
    """OSQP defaults + the reference's overrides (trajopt_sco/src/osqp_interface.cpp:78-90)."""
    s = QpSettings()
    s.rho, s.sigma, s.alpha = 0.1, 1e-6, 1.6
    s.eps_abs, s.eps_rel = 1e-4, 1e-6
    s.eps_prim_inf = s.eps_dual_inf = 1e-4
    s.delta, s.adaptive_rho_tolerance = 1e-6, 5.0
    s.max_iter, s.scaling, s.check_termination = 8192, 10, 25
    s.adaptive_rho, s.adaptive_rho_interval = 1, 50
    s.polishing, s.polish_refine_iter, s.warm_starting = 1, 3, 1
    s.early_polish_every, s.early_polish_from = 25, 25  # optimisation O1 (DESIGN.md); 0 = OSQP's order
    return s


def sqp_table(rows, B):
    """A ctypes array of B SqpParams (the per-trajectory table of tb200_problem_desc.sqp_per_traj) from a sequence."""
    rows = list(rows)
    if len(rows) != B:
        raise ValueError(f"{len(rows)} parameter rows for a batch of {B}")
    return (SqpParams * B)(*rows)


def _dp(a):
    return a.ctypes.data_as(_dbl_p) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(_i32_p) if a is not None else None


class ProblemDesc:
    """Python-side owner of a tb200_problem_desc: keeps every buffer alive."""

    def __init__(self, robot, n_steps, terms, init_traj, fixed_timesteps=(), fixed_dofs=(), cart_targets=None,
                 obstacles=None, obstacles_per_traj=True, sqp=None, qp=None, group_size=0, group_stop=0, sqp_per_traj=None):
        """group_size G >= 2: trajectories [g*G, (g+1)*G) are G seeds of problem g; group_stop 1: the siblings of a seed
        that converges stop at their next SQP iteration top (include/trajopt_b200.h).  sqp_per_traj: B SqpParams, the
        parameters trajectory b runs under (None: `sqp` for every trajectory)."""
        self.robot_spec = robot
        init_traj = np.ascontiguousarray(init_traj, dtype=np.float64)
        assert init_traj.ndim == 3 and init_traj.shape[1] == n_steps and init_traj.shape[2] == robot["n_dof"]
        self.B, self.T, self.D = init_traj.shape
        self.init_traj = init_traj
        self.terms = list(terms)
        self._segs = (Segment * len(robot["segments"]))(*robot["segments"])
        self._lower = np.ascontiguousarray(robot["lower"], dtype=np.float64)
        self._upper = np.ascontiguousarray(robot["upper"], dtype=np.float64)
        sph = robot.get("spheres", [])
        self._spheres = (Sphere * max(len(sph), 1))(*sph)
        self._terms = (Term * max(len(self.terms), 1))(*self.terms)
        self._fixed_t = np.ascontiguousarray(list(fixed_timesteps), dtype=np.int32)
        self._fixed_d = np.ascontiguousarray(list(fixed_dofs), dtype=np.int32)
        self.cart_targets = None if cart_targets is None else np.ascontiguousarray(cart_targets, dtype=np.float64)
        self.obstacles = None if obstacles is None else np.ascontiguousarray(obstacles, dtype=np.float64)
        d = ProblemDescC()
        d.robot.n_dof = robot["n_dof"]
        d.robot.n_segments = len(robot["segments"])
        d.robot.segments = self._segs
        d.robot.lower = _dp(self._lower)
        d.robot.upper = _dp(self._upper)
        d.robot.n_spheres = len(sph)
        d.robot.spheres = self._spheres
        d.n_steps, d.batch, d.n_terms = self.T, self.B, len(self.terms)
        d.terms = self._terms
        d.n_fixed_timesteps = len(self._fixed_t)
        d.fixed_timesteps = _ip(self._fixed_t)
        d.n_fixed_dofs = len(self._fixed_d)
        d.fixed_dofs = _ip(self._fixed_d)
        d.init_traj = _dp(self.init_traj)
        if self.cart_targets is not None:
            assert self.cart_targets.shape[0] == self.B and self.cart_targets.shape[-1] == 7
            d.n_cart_targets = self.cart_targets.shape[1]
            d.cart_targets = _dp(self.cart_targets)
        if self.obstacles is not None:
            d.n_obstacles = self.obstacles.shape[-2]
            d.obstacles_per_traj = 1 if obstacles_per_traj else 0
            d.obstacles = _dp(self.obstacles)
        d.sqp = sqp if sqp is not None else default_sqp_params()
        d.qp = qp if qp is not None else default_qp_settings()
        d.group_size, d.group_stop = group_size, group_stop
        self.sqp_per_traj = None
        if sqp_per_traj is not None:
            self.sqp_per_traj = sqp_table(sqp_per_traj, self.B)
            d.sqp_per_traj = self.sqp_per_traj
        self.c = d

    def slice(self, b0, b1):
        """A description holding only trajectories [b0, b1) (for sharding / small oracle runs).  With groups the cut
        must fall on group boundaries: a group is never split."""
        G = max(self.c.group_size, 1)
        if b0 % G or b1 % G:
            raise ValueError(f"[{b0}, {b1}) splits a group of {G} seeds")
        return ProblemDesc(self.robot_spec, self.T, self.terms, self.init_traj[b0:b1],
                           fixed_timesteps=self._fixed_t, fixed_dofs=self._fixed_d,
                           cart_targets=None if self.cart_targets is None else self.cart_targets[b0:b1],
                           obstacles=None if self.obstacles is None else
                           (self.obstacles[b0:b1] if self.c.obstacles_per_traj else self.obstacles),
                           obstacles_per_traj=bool(self.c.obstacles_per_traj), sqp=self.c.sqp, qp=self.c.qp,
                           group_size=self.c.group_size, group_stop=self.c.group_stop,
                           sqp_per_traj=None if self.sqp_per_traj is None else self.sqp_per_traj[b0:b1])


def alloc_results(B, T, D, n_costs, n_cnts):
    """Caller-owned result buffers (numpy) + the ctypes view."""
    buf = dict(x=np.zeros((B, T, D)), status=np.full(B, OPT_INVALID, np.int32), total_cost=np.zeros(B),
               cost_vals=np.zeros((B, max(n_costs, 1))), cnt_viols=np.zeros((B, max(n_cnts, 1))),
               n_qp_solves=np.zeros(B, np.int32), n_func_evals=np.zeros(B, np.int32),
               n_admm_iters=np.zeros(B, np.int32))
    r = Results()
    r.x, r.total_cost = _dp(buf["x"]), _dp(buf["total_cost"])
    r.cost_vals, r.cnt_viols = _dp(buf["cost_vals"]), _dp(buf["cnt_viols"])
    r.status, r.n_qp_solves = _ip(buf["status"]), _ip(buf["n_qp_solves"])
    r.n_func_evals, r.n_admm_iters = _ip(buf["n_func_evals"]), _ip(buf["n_admm_iters"])
    buf["cost_vals"] = buf["cost_vals"][:, :n_costs]
    buf["cnt_viols"] = buf["cnt_viols"][:, :n_cnts]
    return buf, r


_LIB = None


def library_path():
    if os.environ.get("TB200_LIB"):  # an alternative build of the SAME CUDA library (kernel experiments)
        return os.environ["TB200_LIB"]
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libtrajopt_b200.so")


def load_library():
    """Load the CUDA build of the C ABI.  Raises (never falls back) when it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(the product path is CUDA-only; there is no CPU fallback)")
    lib = C.CDLL(path)
    lib.tb200_version.restype = C.c_char_p
    lib.tb200_last_error.restype = C.c_char_p
    lib.tb200_problem_create.argtypes = [C.POINTER(ProblemDescC), C.c_int, C.POINTER(C.c_void_p)]
    lib.tb200_problem_destroy.argtypes = [C.c_void_p]
    lib.tb200_problem_destroy.restype = None
    lib.tb200_problem_layout.argtypes = [C.c_void_p, C.POINTER(Layout)]
    lib.tb200_problem_set_inputs.argtypes = [C.c_void_p, _dbl_p, _dbl_p, _dbl_p]
    lib.tb200_solve_batch.argtypes = [C.c_void_p, C.POINTER(Results)]
    lib.tb200_solve_batch_resident.argtypes = [C.c_void_p]
    lib.tb200_fetch_results.argtypes = [C.c_void_p, C.POINTER(Results)]
    lib.tb200_convexify_batch.argtypes = [C.c_void_p, _dbl_p, C.POINTER(ConvexifyOut)]
    lib.tb200_qp_solve_batch.argtypes = [C.c_void_p, _dbl_p, _dbl_p, _dbl_p, _dbl_p, _i32_p, _dbl_p, _dbl_p, _i32_p]
    lib.tb200_last_qp_polish.argtypes = [C.c_void_p, _i32_p]
    lib.tb200_last_timing.argtypes = [C.c_void_p, C.POINTER(Timing)]
    lib.tb200_default_sqp_params.argtypes = [C.POINTER(SqpParams)]
    lib.tb200_problem_set_sqp_params.argtypes = [C.c_void_p, C.POINTER(SqpParams)]
    lib.tb200_problem_set_sqp_params_per_traj.argtypes = [C.c_void_p, C.POINTER(SqpParams)]
    lib.tb200_default_qp_settings.argtypes = [C.POINTER(QpSettings)]
    lib.tb200_problem_set_groups.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.tb200_fetch_group_results.argtypes = [C.c_void_p, C.POINTER(GroupResults)]
    lib.tb200_check_trajectories.argtypes = [C.c_void_p, _dbl_p, C.POINTER(CheckConfig), C.POINTER(CheckResults)]
    lib.tb200_problem_set_sqp_log.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.tb200_fetch_sqp_log.argtypes = [C.c_void_p, C.POINTER(SqpLog)]
    lib.tb200_problem_objects.argtypes = [C.c_void_p, _i32_p, _i32_p]
    _LIB = lib
    return lib


EXPORTED_SYMBOLS = [
    "tb200_version", "tb200_last_error", "tb200_default_sqp_params", "tb200_default_qp_settings",
    "tb200_problem_create", "tb200_problem_destroy", "tb200_problem_layout", "tb200_problem_set_inputs",
    "tb200_solve_batch", "tb200_solve_batch_resident", "tb200_fetch_results", "tb200_convexify_batch",
    "tb200_qp_solve_batch", "tb200_last_qp_polish", "tb200_last_timing",
    "tb200_qp_solve_general", "tb200_qp_general_last_error", "tb200_osqp_order_qp_settings", "tb200_problem_set_sqp_params",
    "tb200_problem_set_groups", "tb200_fetch_group_results", "tb200_check_trajectories",
    "tb200_problem_set_sqp_log", "tb200_fetch_sqp_log", "tb200_problem_objects", "tb200_problem_set_sqp_params_per_traj",
]
