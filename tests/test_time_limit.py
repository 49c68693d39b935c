"""The SQP time limit (sco::BasicTrustRegionSQPParameters::max_time, optimizers.cpp:738-753; DESIGN.md section 6).

The limit is checked at the top of every SQP iteration; a trajectory past it ends with its last accepted iterate,
OPT_CONVERGED when it has no constraints or max(cnt_viols) < cnt_tolerance, else OPT_TIME_LIMIT.  The CPU model of it
is the oracle's SQP driver with its wall-clock stop rule (oracle_lib.solve_batch(..., wall_clock=True)); its QP-budget
rule ("stop at the first iteration top with n_qp_solves >= budget") makes a time-limited device run checkable exactly.
CPU: defaults, both JSON readers, the CPU model at max_time 0 / DBL_MAX.  GPU (-m gpu): the device against it."""
import ctypes as C
import json
import subprocess
import sys

import numpy as np
import pytest

import cpp_host
from trajopt_b200 import api, capi, json_io, problems

DBL_MAX = sys.float_info.max
_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "time_limit_host")


def _costs_only(d):
    """The same description without its constraints."""
    terms = [t for t in d.terms if t.role == capi.ROLE_COST]
    return capi.ProblemDesc(d.robot_spec, d.T, terms, d.init_traj, fixed_timesteps=d._fixed_t, fixed_dofs=d._fixed_d,
                            cart_targets=d.cart_targets, obstacles=d.obstacles, obstacles_per_traj=bool(d.c.obstacles_per_traj))


_MAKERS = {"cfg1": lambda: problems.config1(B=8, T=12), "cfg2": lambda: problems.config2(B=8, T=12),
           "cfg3": lambda: problems.config3(B=8, T=12, via_every=4), "variants": lambda: problems.config_variants(B=8, T=10),
           "variants_costs_only": lambda: _costs_only(problems.config_variants(B=4, T=10)),
           "cfg4_short": lambda: problems.config4(B=4, T=12)}


def _with_max_time(d, t):
    d.c.sqp.max_time = t
    return d


def _status_rule(cnt_viols, cnt_tolerance):
    """OPT_CONVERGED when there are no constraints or all are within tolerance, else OPT_TIME_LIMIT."""
    if cnt_viols.shape[-1] == 0:
        return np.full(cnt_viols.shape[0], capi.OPT_CONVERGED)
    return np.where(cnt_viols.max(axis=-1) < cnt_tolerance, capi.OPT_CONVERGED, capi.OPT_TIME_LIMIT)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_default_max_time_is_dbl_max():
    lib = capi.load_library()
    s = capi.SqpParams()
    lib.tb200_default_sqp_params(C.byref(s))
    assert s.max_time == DBL_MAX
    assert bytes(capi.default_sqp_params()) == bytes(s)  # the hand-written Python defaults agree field by field


DOC = {"basic_info": {"n_steps": 6, "manip": "arm"},
       "costs": [{"type": "joint_vel", "params": {"coeffs": [1], "targets": [0]}}],
       "constraints": [{"type": "joint_pos", "params": {"targets": [0.5, 0.5, 0.5], "first_step": 5, "last_step": 5}}],
       "init_info": {"type": "joint_interpolated", "endpoint": [0.2, 0.2, 0.2]}}


def _doc(max_time=None, endpoint=None):
    d = json.loads(json.dumps(DOC))
    if max_time is not None:
        d["opt_info"] = {"max_time": max_time, "max_iter": 30}
    if endpoint is not None:
        d["init_info"]["endpoint"] = endpoint
    return d


def test_python_json_reader_maps_max_time():
    d = problems.config0()
    robot = dict(d.robot_spec)
    doc = {"basic_info": {"n_steps": 5, "manip": "right_arm"},
           "costs": [{"type": "joint_vel", "params": {"coeffs": [1], "targets": [0]}}],
           "init_info": {"type": "stationary"}}
    assert json_io.from_json(doc, robot, np.zeros((1, 7))).c.sqp.max_time == DBL_MAX
    doc["opt_info"] = {"max_time": 0.25}
    assert json_io.from_json(doc, robot, np.zeros((1, 7))).c.sqp.max_time == 0.25


@pytest.mark.parametrize("max_time,want", [(None, "1.7976931348623157e+308"), (0.25, "0.25"), (0, "0")])
def test_cpp_json_reader_maps_max_time(host_bin, tmp_path, max_time, want):
    path = str(tmp_path / "doc.json")
    with open(path, "w") as f:
        json.dump(_doc(max_time), f)
    out = subprocess.run([host_bin, path, "params"], check=True, capture_output=True, text=True).stdout.split()
    assert out == ["max_time", want]


@pytest.mark.parametrize("name", sorted(_MAKERS))
def test_oracle_max_time_zero_stops_after_the_initial_evaluation(oracle, name):
    d = _with_max_time(_MAKERS[name](), 0.0)
    r = oracle.solve_batch(d, wall_clock=True)
    assert (r["n_qp_solves"] == 0).all() and (r["n_func_evals"] == 1).all() and (r["ended"] == 1).all()
    # the closest feasible point of the initial trajectory (modeling.cpp:261-269, including its overwritten lower clip)
    upper = np.asarray(d.robot_spec["upper"], float)
    np.testing.assert_array_equal(r["x"], np.minimum(upper - 1e-3, d.init_traj))
    np.testing.assert_array_equal(r["status"], _status_rule(r["cnt_viols"], d.c.sqp.cnt_tolerance))
    # the values returned are the exact ones at that point
    ref = oracle.convexify_batch(d, r["x"])
    np.testing.assert_array_equal(r["cost_vals"], ref["cost_vals"])
    np.testing.assert_array_equal(r["cnt_viols"], ref["cnt_viols"])
    if name == "variants_costs_only":
        assert (r["status"] == capi.OPT_CONVERGED).all()
    if name in ("cfg2", "cfg3", "cfg4_short"):
        assert (r["status"] == capi.OPT_TIME_LIMIT).any()  # an unoptimised trajectory is not labelled converged


@pytest.mark.parametrize("name", ["cfg1", "cfg2", "variants"])
def test_oracle_without_a_limit_is_the_default_oracle(oracle, name):
    d = _MAKERS[name]()
    ref = oracle.solve_batch(d)
    for t in (DBL_MAX, float("nan"), 1e6):
        r = oracle.solve_batch(_with_max_time(d, t), wall_clock=True)
        assert (r["ended"] == 0).all()
        for k in ("status", "n_qp_solves", "n_func_evals", "n_admm_iters", "x", "total_cost", "cost_vals", "cnt_viols"):
            np.testing.assert_array_equal(r[k], ref[k], err_msg=k)


def test_oracle_negative_max_time_stops_at_the_first_check(oracle):
    d = _with_max_time(_MAKERS["cfg2"](), -1.0)
    r = oracle.solve_batch(d, wall_clock=True)
    assert (r["n_qp_solves"] == 0).all() and (r["ended"] == 1).all()


@pytest.mark.parametrize("name", ["cfg2", "variants"])
def test_oracle_qp_budget_zero_is_max_time_zero(oracle, name):
    d = _MAKERS[name]()
    a = oracle.solve_batch(d, qp_budget=np.zeros(d.B, np.int32))
    b = oracle.solve_batch(_with_max_time(d, 0.0), wall_clock=True)
    for k in ("status", "n_qp_solves", "n_func_evals", "x", "total_cost", "cost_vals", "cnt_viols", "ended"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_oracle_qp_budget_stops_at_an_iteration_top(oracle):
    """A budget of k QPs ends each trajectory at the first iteration top at or after k QPs: the trajectories that need
    fewer are the untimed ones, the others stop after at least k QPs, never more than one SQP iteration later."""
    d = _MAKERS["cfg2"]()
    full = oracle.solve_batch(d)
    k = 3
    r = oracle.solve_batch(d, qp_budget=np.full(d.B, k, np.int32))
    done = full["n_qp_solves"] <= k  # (an untimed run that reaches an iteration top always solves one more QP)
    assert (r["ended"][done] == 0).all()
    for key in ("status", "n_qp_solves", "x", "total_cost"):
        np.testing.assert_array_equal(r[key][done], full[key][done], err_msg=key)
    cut = r["ended"] == 1
    assert cut.any()
    assert (r["n_qp_solves"][cut] >= k).all() and (r["n_qp_solves"][cut] < full["n_qp_solves"][cut]).all()
    np.testing.assert_array_equal(r["status"][cut], _status_rule(r["cnt_viols"][cut], d.c.sqp.cnt_tolerance))


# ---------------------------------------------------------------------------------------------------------------- GPU
def _device_solve(p, trace_cap=0):
    """Solve on an api.Problem; returns results with the decision trace (trace_cap > 0), the "ended by the clock"
    flags, the clock start and the finish time of every trajectory (ns of %globaltimer)."""
    if trace_cap:
        p.lib.tb200_debug_enable_trace(p.handle, trace_cap)
    got = p.solve()
    B = p.desc.B
    if trace_cap:
        tr, tl = np.zeros((B, trace_cap, 14)), np.zeros(B, np.int32)
        p.lib.tb200_debug_fetch_trace(p.handle, tr.ctypes.data_as(_dbl_p), tl.ctypes.data_as(_i32_p))
        got["trace"], got["trace_len"] = tr, tl
    start, ended = C.c_uint64(0), np.zeros(B, np.int32)
    assert p.lib.tb200_debug_time_limit(p.handle, C.byref(start), ended.ctypes.data_as(_i32_p)) == 0
    sched = np.zeros(1 + 2 * B, np.uint64)
    p.lib.tb200_debug_schedule(p.handle, sched.ctypes.data_as(C.POINTER(C.c_uint64)))
    got["ended"], got["clock_start"], got["finish_ns"] = ended, start.value, sched[1:1 + B]
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_MAKERS))
def test_device_max_time_zero_matches_oracle(oracle, name):
    d = _with_max_time(_MAKERS[name](), 0.0)
    p = api.Problem(d)
    got = _device_solve(p)
    p.close()
    ref = oracle.solve_batch(d, wall_clock=True)
    assert (got["ended"] == 1).all()
    for k in ("status", "n_qp_solves", "n_func_evals", "x"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    assert (got["n_qp_solves"] == 0).all() and (got["n_func_evals"] == 1).all()
    np.testing.assert_allclose(got["cost_vals"], ref["cost_vals"], rtol=1e-12, atol=1e-14)  # test_convexify_rows_match_oracle
    np.testing.assert_allclose(got["cnt_viols"], ref["cnt_viols"], rtol=1e-9, atol=1e-12)
    np.testing.assert_array_equal(got["status"], _status_rule(got["cnt_viols"], d.c.sqp.cnt_tolerance))


@pytest.mark.gpu
def test_device_explicit_no_limit_is_bitwise_the_default():
    d = problems.config2(B=64, T=30)
    p = api.Problem(d)
    base = p.solve()
    for t in (DBL_MAX, 1e6):
        sqp = capi.default_sqp_params()
        sqp.max_time = t
        p.set_sqp_params(sqp)
        got = _device_solve(p)
        assert (got["ended"] == 0).all()
        for k in ("status", "n_qp_solves", "n_func_evals", "n_admm_iters", "x", "total_cost", "cost_vals", "cnt_viols"):
            np.testing.assert_array_equal(got[k], base[k], err_msg=f"{k} (max_time {t})")
    p.close()


def _unverified(tr, tl, qp_max_iter):
    """_solve_with_trace's rule (tests/test_gpu_parity.py): a QP that hit the iteration limit or ended without a
    KKT-verified polish makes a trajectory incomparable step by step."""
    return np.array([(tr[b, :tl[b], 7] >= qp_max_iter).any() or (tr[b, :tl[b], 12] != 1).any() for b in range(len(tl))])


@pytest.mark.gpu
@pytest.mark.parametrize("name,make", [("cfg2", lambda: problems.config2(B=256, T=30)),
                                       ("cfg3", lambda: problems.config3(B=32, T=30))])
def test_device_intermediate_budget(oracle, name, make):
    d = make()
    cap = 600
    p = api.Problem(d)
    full = _device_solve(p, cap)
    assert (full["ended"] == 0).all()
    finish_s = (full["finish_ns"].astype(np.int64) - np.int64(full["clock_start"])) * 1e-9
    budget = float(np.median(finish_s))
    sqp = capi.default_sqp_params()
    sqp.max_time = budget
    p.set_sqp_params(sqp)
    lim = _device_solve(p, cap)
    p.close()
    tf, lf, tl, ll = full["trace"], full["trace_len"], lim["trace"], lim["trace_len"]
    # every trajectory's decisions are a bitwise prefix of its untimed ones
    assert (ll <= lf).all()
    for b in range(d.B):
        np.testing.assert_array_equal(tl[b, :ll[b]], tf[b, :ll[b]], err_msg=f"trajectory {b}")
    cut = ll < lf
    np.testing.assert_array_equal(lim["ended"], cut.astype(np.int32))
    assert cut.any() and (~cut).any(), (budget, ll, lf)
    for k in ("status", "n_qp_solves", "n_func_evals", "n_admm_iters", "x", "total_cost", "cost_vals", "cnt_viols"):
        np.testing.assert_array_equal(lim[k][~cut], full[k][~cut], err_msg=k)
    assert (lim["n_qp_solves"][cut] == ll[cut]).all()
    # stopped at an iteration top: the untimed run's next QP starts a new (merit round, iteration)
    for b in np.nonzero(cut)[0]:
        n = ll[b]
        assert n == 0 or tuple(tf[b, n, :2]) != tuple(tf[b, n - 1, :2]), (b, tf[b, max(n - 1, 0):n + 1, :2])
    np.testing.assert_array_equal(lim["status"][cut], _status_rule(lim["cnt_viols"][cut], d.c.sqp.cnt_tolerance))
    # against the CPU model with the device's QP counts as budgets, where every QP was KKT-verified
    ok = ~_unverified(tl, ll, d.c.qp.max_iter)
    assert ok.mean() >= 0.75
    ref = oracle.solve_batch(d, qp_budget=lim["n_qp_solves"])
    np.testing.assert_array_equal(lim["status"][ok], ref["status"][ok])
    np.testing.assert_array_equal(lim["n_qp_solves"][ok], ref["n_qp_solves"][ok])
    np.testing.assert_allclose(lim["total_cost"][ok], ref["total_cost"][ok], atol=1e-6)
    assert lim["timing"]["total_ms"] < full["timing"]["total_ms"]


@pytest.mark.gpu
@pytest.mark.parametrize("endpoint", [[0.2, 0.2, 0.2], [0.5, 0.5, 0.5]])
def test_cpp_host_layer_max_time_zero(host_bin, tmp_path, endpoint):
    """ConstructProblem + OptimizeWithParams with opt_info.max_time = 0: no QP, and the status rule (the joint_pos
    constraint is violated by the initial trajectory of the first endpoint and met by the second)."""
    path = str(tmp_path / "doc.json")
    with open(path, "w") as f:
        json.dump(_doc(0, endpoint), f)
    out = subprocess.run([host_bin, path, "solve"], check=True, capture_output=True, text=True).stdout.splitlines()
    assert len(out) == 2
    want = capi.OPT_TIME_LIMIT if endpoint[0] != 0.5 else capi.OPT_CONVERGED
    for line in out:
        status, nqp, nfe, n_cnts, mx, tol = line.split()
        assert int(nqp) == 0 and int(nfe) == 1 and int(n_cnts) == 1
        assert int(status) == (capi.OPT_CONVERGED if float(mx) < float(tol) else capi.OPT_TIME_LIMIT) == want
