"""Loader for the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE: imported only by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg."""
import ctypes as C
import os
import subprocess

import numpy as np

from trajopt_b200 import capi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


def build():
    subprocess.run(["make", "-C", os.path.join(_ROOT, "oracle"), "-s"], check=True)


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_ROOT, "oracle", "liboracle.so")
        if not os.path.exists(path):
            build()
        _LIB = C.CDLL(path)
        _LIB.oracle_last_error.restype = C.c_char_p
        _LIB.oracle_quad_value.restype = C.c_double
    return _LIB


def _dp(a):
    return a.ctypes.data_as(_dbl_p) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(_i32_p) if a is not None else None


def layout(desc):
    L = capi.Layout()
    rc = lib().oracle_layout(C.byref(desc.c), C.byref(L))
    assert rc == 0, lib().oracle_last_error()
    return L


class Records(C.Structure):
    """oracle_records (oracle/capi.cpp): the iteration log of every trajectory, [B][cap][...]."""
    _fields_ = [("cap", C.c_int), ("n", _i32_p)] + [(k, _dbl_p) for k in (
        "trace", "merit_coeffs", "model_cost_vals", "model_cnt_viols", "cost_vals", "cnt_viols", "x")]


STOP_NONE, STOP_WALL_CLOCK, STOP_QP_BUDGET = 0, 1, 2


def solve_batch(desc, b0=0, b1=None, n_threads=0, trace_b=-1, wall_clock=False, qp_budget=None, records=0):
    """The oracle's SQP on trajectories [b0, b1).  Returns the result buffers plus "seconds" (wall time of the call),
    "ended" ([B], 1 where the stop rule ended the trajectory) and "trace" (the decision trace of trajectory trace_b).
    Stop rule: wall_clock, a steady clock per trajectory against desc.c.sqp.max_time (which is not read otherwise), or
    qp_budget ([B] ints), stop at the first iteration top with n_qp_solves >= qp_budget[b].  records > 0: also "log",
    up to that many records per trajectory (record 0 the start, then one per QP solve; unwritten entries NaN)."""
    b1 = desc.B if b1 is None else b1
    L = layout(desc)
    buf, res = capi.alloc_results(desc.B, desc.T, desc.D, L.n_costs, L.n_cnts)
    buf["ended"] = np.zeros(desc.B, np.int32)
    secs = C.c_double(0)
    if not wall_clock and qp_budget is None and not records:
        trace = np.zeros((4096, 14))
        tlen = C.c_int(0)
        rc = lib().oracle_solve_batch(C.byref(desc.c), b0, b1, n_threads, C.byref(res), C.byref(secs), trace_b,
                                      _dp(trace), 4096, C.byref(tlen))
        assert rc == 0, lib().oracle_last_error()
        buf["seconds"] = secs.value
        buf["trace"] = trace[:tlen.value]
        return buf
    stop, budget = STOP_NONE, None
    if qp_budget is not None:
        stop, budget = STOP_QP_BUDGET, np.ascontiguousarray(np.broadcast_to(qp_budget, (desc.B,)), dtype=np.int32)
    elif wall_clock:
        stop = STOP_WALL_CLOCK
    cap = max(records, 4097 if trace_b >= 0 else 0)
    rec, log = None, None
    if cap:
        B, nc, nk = desc.B, L.n_costs, L.n_cnts
        log = dict(n_records=np.zeros(B, np.int32), trace=np.full((B, cap, 14), np.nan))
        if records:
            log.update(mu=np.full((B, cap, nk), np.nan), model_cost_vals=np.full((B, cap, nc), np.nan),
                       model_cnt_viols=np.full((B, cap, nk), np.nan), new_cost_vals=np.full((B, cap, nc), np.nan),
                       new_cnt_viols=np.full((B, cap, nk), np.nan), x=np.full((B, cap, desc.T * desc.D), np.nan))
        arr = [_dp(log[k]) if k in log and log[k].size else None for k in
               ("trace", "mu", "model_cost_vals", "model_cnt_viols", "new_cost_vals", "new_cnt_viols", "x")]
        rec = Records(cap, _ip(log["n_records"]), *arr)
    rc = lib().oracle_solve_batch_ext(C.byref(desc.c), b0, b1, n_threads, stop, _ip(budget), C.byref(res),
                                      _ip(buf["ended"]), None if rec is None else C.byref(rec), C.byref(secs))
    assert rc == 0, lib().oracle_last_error()
    buf["seconds"] = secs.value
    buf["trace"] = log["trace"][trace_b, 1:log["n_records"][trace_b]] if trace_b >= 0 else np.zeros((0, 14))
    if records:
        buf["log"] = log
    return buf


def objects(desc):
    """(term, step) of every object in OptProb order, as Problem.objects() lists them on the device."""
    L = layout(desc)
    term, step = np.zeros(L.n_costs + L.n_cnts, np.int32), np.zeros(L.n_costs + L.n_cnts, np.int32)
    rc = lib().oracle_objects(C.byref(desc.c), _ip(term), _ip(step))
    assert rc == 0, lib().oracle_last_error()
    return term, step


def sing_svd_min(J):
    """The avoid_singularity term's SVD: sigma, u[6], v[D] of a 6 x D matrix."""
    J = np.ascontiguousarray(J, dtype=np.float64)
    s, u, v = C.c_double(0), np.zeros(6), np.zeros(J.shape[1])
    assert lib().oracle_sing_svd_min(_dp(J), J.shape[1], C.byref(s), _dp(u), _dp(v)) == 0
    return s.value, u, v


def sing_err_grad(desc, q, link, lam):
    """The avoid_singularity term at one waypoint: the Jacobian [6][D], sigma, err and the unscaled gradient."""
    q = np.ascontiguousarray(q, dtype=np.float64)
    J, s, e, g = np.zeros((6, q.size)), C.c_double(0), C.c_double(0), np.zeros(q.size)
    rc = lib().oracle_sing_err_grad(C.byref(desc.c.robot), _dp(q), link, C.c_double(lam), _dp(J), C.byref(s),
                                    C.byref(e), _dp(g))
    assert rc == 0, lib().oracle_last_error()
    return J, s.value, e.value, g


def convexify_batch(desc, x, b0=0, b1=None):
    b1 = desc.B if b1 is None else b1
    L = layout(desc)
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = dict(cart_err=np.zeros((desc.B, max(L.n_cart_rows, 1))),
               cart_jac=np.zeros((desc.B, max(L.n_cart_rows, 1), max(L.cart_jac_stride, 1))),
               coll_rows=np.zeros((desc.B, max(L.n_coll_cand, 1), L.coll_row_stride)),
               cost_vals=np.zeros((desc.B, max(L.n_costs, 1))), cnt_viols=np.zeros((desc.B, max(L.n_cnts, 1))))
    co = capi.ConvexifyOut(*[_dp(out[k]) for k in ("cart_err", "cart_jac", "coll_rows", "cost_vals", "cnt_viols")])
    rc = lib().oracle_convexify_batch(C.byref(desc.c), b0, b1, _dp(x), C.byref(co))
    assert rc == 0, lib().oracle_last_error()
    out["cart_err"] = out["cart_err"][:, :L.n_cart_rows]
    out["cart_jac"] = out["cart_jac"][:, :L.n_cart_rows]
    out["coll_rows"] = out["coll_rows"][:, :L.n_coll_cand]
    out["cost_vals"] = out["cost_vals"][:, :L.n_costs]
    out["cnt_viols"] = out["cnt_viols"][:, :L.n_cnts]
    return out


def qp_solve_batch(desc, x, trust, merit_coeffs, b0=0, b1=None):
    b1 = desc.B if b1 is None else b1
    L = layout(desc)
    x = np.ascontiguousarray(x, dtype=np.float64)
    trust = np.ascontiguousarray(np.broadcast_to(trust, (desc.B,)), dtype=np.float64)
    mc = np.ascontiguousarray(np.broadcast_to(merit_coeffs, (desc.B, max(L.n_cnts, 1))), dtype=np.float64)
    out = dict(new_x=np.zeros((desc.B, desc.T, desc.D)), qp_status=np.zeros(desc.B, np.int32),
               model_cost_vals=np.zeros((desc.B, max(L.n_costs, 1))), model_cnt_viols=np.zeros((desc.B, max(L.n_cnts, 1))),
               admm_iters=np.zeros(desc.B, np.int32), kkt=np.zeros((desc.B, 3)), polish=np.zeros(desc.B, np.int32))
    rc = lib().oracle_qp_solve_batch(C.byref(desc.c), b0, b1, _dp(x), _dp(trust), _dp(mc), _dp(out["new_x"]),
                                     _ip(out["qp_status"]), _dp(out["model_cost_vals"]), _dp(out["model_cnt_viols"]),
                                     _ip(out["admm_iters"]), _dp(out["kkt"]), _ip(out["polish"]))
    assert rc == 0, lib().oracle_last_error()
    out["model_cost_vals"] = out["model_cost_vals"][:, :L.n_costs]
    out["model_cnt_viols"] = out["model_cnt_viols"][:, :L.n_cnts]
    return out
