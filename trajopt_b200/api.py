"""Python host layer over the C ABI (include/trajopt_b200.h).  CUDA only: `Problem` raises when the
library is missing or no device is visible — there is no CPU fallback (the CPU oracle lives under oracle/
and is test infrastructure)."""
import ctypes as C

import numpy as np

from . import capi

_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


def _dp(a):
    return a.ctypes.data_as(_dbl_p)


def _ip(a):
    return a.ctypes.data_as(_i32_p)


class Problem:
    """Owns a tb200_problem handle (device buffers for one batched description)."""

    def __init__(self, desc, device=0):
        self.lib = capi.load_library()
        self.desc = desc
        self.handle = C.c_void_p()
        rc = self.lib.tb200_problem_create(C.byref(desc.c), device, C.byref(self.handle))
        if rc != 0:
            raise RuntimeError(f"tb200_problem_create failed ({rc}): {self.lib.tb200_last_error().decode()}")
        self.layout = capi.Layout()
        self._check(self.lib.tb200_problem_layout(self.handle, C.byref(self.layout)))
        self.group_size = max(desc.c.group_size, 1)
        self._solved_group_size = None
        self._log_shape = (0, False)
        self._solved_log_shape = None

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"trajopt_b200 error {rc}: {self.lib.tb200_last_error().decode()}")

    def close(self):
        if self.handle:
            self.lib.tb200_problem_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_inputs(self, init_traj=None, cart_targets=None, obstacles=None):
        def ptr(a):
            return None if a is None else _dp(np.ascontiguousarray(a, dtype=np.float64))
        keep = [np.ascontiguousarray(a, dtype=np.float64) if a is not None else None for a in (init_traj, cart_targets, obstacles)]
        self._check(self.lib.tb200_problem_set_inputs(self.handle, *[None if a is None else _dp(a) for a in keep]))

    def set_sqp_params(self, sqp):
        """Replace the optimizer parameters for the next solves: one capi.SqpParams (e.g. with a new max_time) for every
        trajectory, or a sequence of B of them, row b for trajectory b (None: drop such a table; the last uniform
        parameters apply again)."""
        if sqp is None:
            self._check(self.lib.tb200_problem_set_sqp_params_per_traj(self.handle, None))
        elif isinstance(sqp, capi.SqpParams):
            self._check(self.lib.tb200_problem_set_sqp_params(self.handle, C.byref(sqp)))
        else:
            rows = capi.sqp_table(sqp, self.desc.B)
            self._check(self.lib.tb200_problem_set_sqp_params_per_traj(self.handle, rows))

    def set_groups(self, group_size, group_stop=0):
        """Multi-start: trajectories [g*G, (g+1)*G) are G seeds of problem g (G = 0 or 1: no groups); group_stop 1
        ends the siblings of a seed that converges at their next SQP iteration top.  For the next solves."""
        self._check(self.lib.tb200_problem_set_groups(self.handle, group_size, group_stop))
        self.group_size = max(int(group_size), 1)

    def group_results(self):
        """Per group of the last solve: the best seed's batch index, status, total cost and x, and how many seeds
        converged; per trajectory: ended_by (0 its own SQP, 1 the time limit, 2 its group)."""
        d = self.desc
        NG = d.B // (self._solved_group_size or 1)  # (before any solve the library refuses)
        out = dict(best=np.zeros(NG, np.int32), status=np.zeros(NG, np.int32), total_cost=np.zeros(NG),
                   x=np.zeros((NG, d.T, d.D)), n_converged=np.zeros(NG, np.int32), ended_by=np.zeros(d.B, np.int32))
        r = capi.GroupResults(_ip(out["best"]), _ip(out["status"]), _dp(out["total_cost"]), _dp(out["x"]),
                              _ip(out["n_converged"]), _ip(out["ended_by"]))
        self._check(self.lib.tb200_fetch_group_results(self.handle, C.byref(r)))
        return out

    def set_sqp_log(self, capacity, with_x=False):
        """Record the SQP iteration log of the next solves: up to `capacity` records per trajectory (the state after the
        initial evaluation, then one per QP solve), each with its point when with_x.  capacity 0 turns it off."""
        self._check(self.lib.tb200_problem_set_sqp_log(self.handle, int(capacity), 1 if with_x else 0))
        self._log_shape = (int(capacity), bool(with_x))

    def sqp_log(self):
        """The SQP iteration log of the last solve as a dict of numpy arrays (fields of tb200_sqp_log, [B][R](...)).
        Per-record arrays hold NaN / 0 / -1 past n_records[b]; new_x is present only for a log recorded with x."""
        L, d = self.layout, self.desc
        R, with_x = self._solved_log_shape or (0, False)
        B, nc, nk = d.B, L.n_costs, L.n_cnts
        out = dict(n_records=np.zeros(B, np.int32), n_dropped=np.zeros(B, np.int32))
        for k in ("kind", "merit_round", "iter", "qp_status", "admm_iters", "polish", "action", "ended"):
            out[k] = np.zeros((B, R), np.int32)
        for k in ("trust_box_size", "old_merit", "model_merit", "new_merit"):
            out[k] = np.zeros((B, R))
        out["qp_diag"] = np.zeros((B, R, 4))
        out["merit_coeffs"] = np.zeros((B, R, nk))
        for k, n in (("model_cost_vals", nc), ("model_cnt_viols", nk), ("old_cost_vals", nc), ("old_cnt_viols", nk),
                     ("new_cost_vals", nc), ("new_cnt_viols", nk)):
            out[k] = np.zeros((B, R, n))
        if with_x:
            out["new_x"] = np.zeros((B, R, d.T, d.D))
        r = capi.SqpLog(*[(_ip if out[k].dtype == np.int32 else _dp)(out[k]) if k in out and out[k].size else None
                          for k, _ in capi.SqpLog._fields_])
        self._check(self.lib.tb200_fetch_sqp_log(self.handle, C.byref(r)))
        return out

    def objects(self):
        """Per cost / constraint object (costs, then constraints, the order of cost_vals / cnt_viols): the index of
        the term that hatched it and its step."""
        n = self.layout.n_costs + self.layout.n_cnts
        term, step = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        self._check(self.lib.tb200_problem_objects(self.handle, _ip(term), _ip(step)))
        return term[:n], step[:n]

    def _results(self):
        L, d = self.layout, self.desc
        return capi.alloc_results(d.B, d.T, d.D, L.n_costs, L.n_cnts)

    def solve(self):
        """BasicTrustRegionSQP::optimize() for the whole batch; host buffers in and out."""
        buf, res = self._results()
        self._solved_group_size = self.group_size
        self._solved_log_shape = self._log_shape
        self._check(self.lib.tb200_solve_batch(self.handle, C.byref(res)))
        buf["timing"] = self.timing()
        return buf

    def solve_resident(self):
        self._solved_group_size = self.group_size
        self._solved_log_shape = self._log_shape
        self._check(self.lib.tb200_solve_batch_resident(self.handle))

    def fetch(self):
        buf, res = self._results()
        self._check(self.lib.tb200_fetch_results(self.handle, C.byref(res)))
        buf["timing"] = self.timing()
        return buf

    def timing(self):
        t = capi.Timing()
        self._check(self.lib.tb200_last_timing(self.handle, C.byref(t)))
        return {k: getattr(t, k) for k, _ in capi.Timing._fields_}

    def check(self, x=None, type=capi.COLL_DISCRETE, lvs=0.005, margin=0.0):
        """Collision check of every trajectory (tesseract's checkTrajectory): x [B][T][D], or None for the x of the last
        solve (already on the device).  type: capi.COLL_*; lvs: longest valid segment length of the LVS types; margin:
        a contact is a (sphere, obstacle) pair closer than it.  Returns, per slot (S = T for DISCRETE, else T - 1),
        step_min_distance [B][S], step_contacts [B][S] and step_argmin [B][S][3] (sphere, obstacle, sub-index), and per
        trajectory in_collision [B] (bool), first_slot [B] (-1: none) and min_distance [B]."""
        d = self.desc
        S = d.T if type == capi.COLL_DISCRETE else max(d.T - 1, 0)
        out = dict(step_min_distance=np.zeros((d.B, S)), step_contacts=np.zeros((d.B, S), np.int32),
                   step_argmin=np.zeros((d.B, S, 3), np.int32), in_collision=np.zeros(d.B, np.int32),
                   first_slot=np.zeros(d.B, np.int32), min_distance=np.zeros(d.B))
        r = capi.CheckResults(*[(_ip if v.dtype == np.int32 else _dp)(v) if v.size else None for v in out.values()])
        cfg = capi.CheckConfig(type, 0, lvs, margin)
        xp = None
        if x is not None:
            x = np.ascontiguousarray(x, dtype=np.float64)
            if x.shape != (d.B, d.T, d.D):
                raise ValueError(f"x has shape {x.shape}, expected {(d.B, d.T, d.D)}")
            xp = _dp(x)
        self._check(self.lib.tb200_check_trajectories(self.handle, xp, C.byref(cfg), C.byref(r)))
        out["in_collision"] = out["in_collision"].astype(bool)
        return out

    def convexify(self, x):
        L, d = self.layout, self.desc
        x = np.ascontiguousarray(x, dtype=np.float64)
        out = dict(cart_err=np.zeros((d.B, max(L.n_cart_rows, 1))),
                   cart_jac=np.zeros((d.B, max(L.n_cart_rows, 1), max(L.cart_jac_stride, 1))),
                   coll_rows=np.zeros((d.B, max(L.n_coll_cand, 1), L.coll_row_stride)),
                   cost_vals=np.zeros((d.B, max(L.n_costs, 1))), cnt_viols=np.zeros((d.B, max(L.n_cnts, 1))))
        co = capi.ConvexifyOut(*[_dp(out[k]) if n else None for k, n in
                                 (("cart_err", L.n_cart_rows), ("cart_jac", L.n_cart_rows), ("coll_rows", L.n_coll_cand),
                                  ("cost_vals", L.n_costs), ("cnt_viols", L.n_cnts))])
        self._check(self.lib.tb200_convexify_batch(self.handle, _dp(x), C.byref(co)))
        out["cart_err"] = out["cart_err"][:, :L.n_cart_rows]
        out["cart_jac"] = out["cart_jac"][:, :L.n_cart_rows]
        out["coll_rows"] = out["coll_rows"][:, :L.n_coll_cand]
        out["cost_vals"] = out["cost_vals"][:, :L.n_costs]
        out["cnt_viols"] = out["cnt_viols"][:, :L.n_cnts]
        return out

    def convexify_timed(self, x):
        """One full-batch launch of the convexify kernel at `x` without fetching its rows; returns the device
        time (CUDA events on the launching stream) and the algorithmic bytes of the launch."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        co = capi.ConvexifyOut(None, None, None, None, None)
        self._check(self.lib.tb200_convexify_batch(self.handle, _dp(x), C.byref(co)))
        return self.timing()

    def qp_solve(self, x, trust, merit_coeffs):
        L, d = self.layout, self.desc
        x = np.ascontiguousarray(x, dtype=np.float64)
        trust = np.ascontiguousarray(np.broadcast_to(trust, (d.B,)), dtype=np.float64)
        mc = np.ascontiguousarray(np.broadcast_to(merit_coeffs, (d.B, max(L.n_cnts, 1))), dtype=np.float64)
        out = dict(new_x=np.zeros((d.B, d.T, d.D)), qp_status=np.zeros(d.B, np.int32),
                   model_cost_vals=np.zeros((d.B, max(L.n_costs, 1))), model_cnt_viols=np.zeros((d.B, max(L.n_cnts, 1))),
                   admm_iters=np.zeros(d.B, np.int32))
        self._check(self.lib.tb200_qp_solve_batch(self.handle, _dp(x), _dp(trust), _dp(mc), _dp(out["new_x"]),
                                                  _ip(out["qp_status"]), _dp(out["model_cost_vals"]) if L.n_costs else None,
                                                  _dp(out["model_cnt_viols"]) if L.n_cnts else None, _ip(out["admm_iters"])))
        out["model_cost_vals"] = out["model_cost_vals"][:, :L.n_costs]
        out["model_cnt_viols"] = out["model_cnt_viols"][:, :L.n_cnts]
        out["polish"] = np.zeros(d.B, np.int32)
        self._check(self.lib.tb200_last_qp_polish(self.handle, _ip(out["polish"])))
        return out


def solve(desc, device=0, group_size=None, group_stop=None, sqp_log=None, sqp_log_x=False):
    """One-shot: create, solve, destroy.  With group_size (and group_stop) the solve is a multi-start one
    (Problem.set_groups; None keeps the description's own settings) and the result gains a "groups" dict
    (Problem.group_results).  With sqp_log = capacity the SQP iteration log is recorded (with the points when
    sqp_log_x) and the result gains a "sqp_log" dict (Problem.sqp_log)."""
    p = Problem(desc, device)
    try:
        if group_size is not None or group_stop is not None:
            p.set_groups(desc.c.group_size if group_size is None else group_size,
                         desc.c.group_stop if group_stop is None else group_stop)
        if sqp_log:
            p.set_sqp_log(sqp_log, with_x=sqp_log_x)
        out = p.solve()
        if group_size is not None:
            out["groups"] = p.group_results()
        if sqp_log:
            out["sqp_log"] = p.sqp_log()
        return out
    finally:
        p.close()


def check(desc, x, type=capi.COLL_DISCRETE, lvs=0.005, margin=0.0, device=0):
    """One-shot collision check of the trajectories x [B][T][D] against desc's robot and obstacles (Problem.check)."""
    p = Problem(desc, device)
    try:
        return p.check(x, type=type, lvs=lvs, margin=margin)
    finally:
        p.close()


def qp_solve_general(P, q, A, l, u, settings=None, device=0):
    """One sco::Model::optimize() worth of QP on the GPU: min 1/2 x'Px + q'x s.t. l <= Ax <= u (dense inputs; a leading
    batch dimension is allowed).  Returns dict(x, y, status, iters, polish) with OSQP's status values."""
    lib = capi.load_library()
    P = np.ascontiguousarray(P, dtype=np.float64)
    batched = P.ndim == 3
    if not batched:
        P, q, A, l, u = (np.asarray(a, dtype=np.float64)[None] for a in (P, q, A, l, u))
    P, q, A, l, u = (np.ascontiguousarray(a, dtype=np.float64) for a in (P, q, A, l, u))
    B, n = q.shape
    m = l.shape[1]
    g = capi.QpGeneral(n, m, B, 0, _dp(P), _dp(q), _dp(A) if m else None, _dp(l) if m else None, _dp(u) if m else None)
    x, y = np.zeros((B, n)), np.zeros((B, max(m, 1)))
    status, iters, polish = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.int32)
    rc = lib.tb200_qp_solve_general(C.byref(g), C.byref(settings) if settings is not None else None, device, _dp(x), _dp(y),
                                    _ip(status), _ip(iters), _ip(polish))
    if rc != 0:
        lib.tb200_qp_general_last_error.restype = C.c_char_p
        raise RuntimeError(f"tb200_qp_solve_general failed ({rc}): {lib.tb200_qp_general_last_error().decode()}")
    out = dict(x=x, y=y[:, :m], status=status, iters=iters, polish=polish)
    return out if batched else {k: v[0] for k, v in out.items()}
