"""The sco::Model plugin surface (include/trajopt_b200_sco.hpp over tb200_qp_solve_general): the reference's
solver-interface-unit.cpp cases (trajopt_sco/test/solver-interface-unit.cpp:33-73, 136-237) compiled against the header
exactly as they are written against trajopt_sco.  CPU: the canonical QP the model assembles (OSQPModel::updateObjective /
updateConstraints, osqp_interface.cpp:170-281) and its bookkeeping.  GPU: the cases solved, and the general QP entry
point against the CPU oracle's OSQP-equivalent solver on random QPs."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import cpp_host


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "sco_model")


def test_model_assembles_the_canonical_qp(exe):
    """setup_problem: objective (v0 + v1 + v2 - 3)^2, bounds [0, 10]: P = M + M' of exprSquare (diagonal 2, off-diagonal
    2), q = -6, A = I (no constraint rows), l = 0, u = 10; removeVar + update leaves 2 variables; a quadratic inequality
    throws NOT IMPLEMENTED like OSQPModel (osqp_interface.cpp:150)."""
    out = subprocess.run([exe, "dump"], check=True, capture_output=True, text=True).stdout.strip().split("\n")
    n, m = map(int, out[0].split())
    assert (n, m) == (3, 3)
    vec = lambda s: np.array(list(map(float, s.split())))
    np.testing.assert_array_equal(vec(out[1]).reshape(3, 3), 2.0 * np.ones((3, 3)))
    np.testing.assert_array_equal(vec(out[2]), [-6.0, -6.0, -6.0])
    np.testing.assert_array_equal(vec(out[3]).reshape(3, 3), np.eye(3))
    np.testing.assert_array_equal(vec(out[4]), [0.0, 0.0, 0.0])
    np.testing.assert_array_equal(vec(out[5]), [10.0, 10.0, 10.0])
    assert out[6].strip() == "2"
    assert out[7].strip() == "NOT IMPLEMENTED"


@pytest.mark.gpu
def test_reference_solver_interface_cases(exe, tmp_path):
    out = subprocess.run([exe, "solve"], check=True, capture_output=True, text=True, cwd=tmp_path).stdout
    lines = {l.split()[0]: l.split() for l in out.strip().split("\n")}
    assert lines["setup_problem"][2] == "0" and abs(float(lines["setup_problem"][4])) < 1e-6, out  # EXPECT_NEAR(aff.value, 0, 1e-6)
    assert lines["vars_after_remove"][1] == "2"
    assert abs(float(lines["ExprMult_test2"][1]) - 400.0) < 1e-6, out
    assert abs(float(lines["ExprMult_test3"][1]) - 945.0) < 1e-6, out
    assert lines["infeasible"][2] == "1", out  # CVX_INFEASIBLE


@pytest.mark.gpu
def test_general_qp_matches_oracle(oracle):
    """Random strictly convex QPs with equality, inequality and box rows through tb200_qp_solve_general against the
    oracle's OSQP-equivalent solver (oracle_qp_dense): same status, x within 1e-6."""
    from trajopt_b200 import api, capi
    rng = np.random.default_rng(5)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    for n, me, mi in ((4, 1, 2), (12, 3, 6), (40, 5, 30), (90, 10, 60)):
        G = rng.standard_normal((n, n))
        P = G @ G.T / n + 0.1 * np.eye(n)
        q = rng.standard_normal(n)
        x0 = rng.uniform(-0.5, 0.5, n)
        Ae, Ai = rng.standard_normal((me, n)), rng.standard_normal((mi, n))
        A = np.vstack([Ae, Ai, np.eye(n)])
        l = np.concatenate([Ae @ x0, np.full(mi, -1e30), np.full(n, -1.0)])
        u = np.concatenate([Ae @ x0, Ai @ x0 + rng.uniform(0.0, 0.5, mi), np.full(n, 1.0)])
        got = api.qp_solve_general(P, q, A, l, u)
        m = len(l)
        x, y = np.zeros(n), np.zeros(m)
        status, iters, polish = C.c_int(0), C.c_int(0), C.c_int(0)
        st = capi.default_qp_settings()
        assert oracle.lib().oracle_qp_dense(n, m, dp(np.ascontiguousarray(P)), dp(q), dp(np.ascontiguousarray(A)), dp(l), dp(u),
                                            C.byref(st), dp(x), dp(y), C.byref(status), C.byref(iters), C.byref(polish)) == 0
        assert got["status"] == status.value == 1, (n, got["status"], status.value)
        np.testing.assert_allclose(got["x"], x, atol=1e-6)
        # KKT: stationarity of the returned primal / dual pair
        r = P @ got["x"] + q + A.T @ got["y"]
        assert np.abs(r).max() < 1e-5, np.abs(r).max()
