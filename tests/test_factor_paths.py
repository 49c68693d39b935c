"""The cyclic-reduction factorisation with warp-local block inversions (blocks of <= 16 with the factor in shared memory:
the polish system of every layout, and the ADMM system where the partition-inverse form does not fit) against the
CTA-wide one, which TB200_GENERIC_QP_PASSES=1 (read when a problem is created) selects.  Both compute every value by the
same expression in the same order, so the results must be bit for bit the same: any reordered multiply-add of an
inversion moves the factor in its last bits, and the ADMM iterates, iteration counts and polished points with it.
-m gpu."""
import numpy as np
import pytest

from test_shape_sweep import DESCS
from trajopt_b200 import api, problems

pytestmark = pytest.mark.gpu

DESC = {
    "cfg1": lambda: problems.config1(B=32, T=30),
    "cfg2": lambda: problems.config2(B=32, T=30),
    "cfg3": lambda: problems.config3(B=16, T=50),
    # 6, 3 and 2 joints (blocks of 12, 6 and 4) at lengths where the ADMM system takes the cyclic reduction too
    "d6_T33": lambda: DESCS["d6_T33"],
    "d3_T64": lambda: DESCS["d3_T64"],
    "d2_T40": lambda: DESCS["d2_T40"],
}


def _both(monkeypatch, desc, run):
    out = []
    for generic in ("1", "0"):
        monkeypatch.setenv("TB200_GENERIC_QP_PASSES", generic)
        p = api.Problem(desc)
        try:
            out.append(run(p))
        finally:
            p.close()
    return out


@pytest.mark.parametrize("name", list(DESC))
@pytest.mark.parametrize("trust", [0.1, 0.01])
def test_qp_solve_factor_paths_identical(monkeypatch, name, trust):
    d = DESC[name]()
    x = d.init_traj.copy()
    cta, warp = _both(monkeypatch, d, lambda p: p.qp_solve(x, trust, 10.0))
    for k in ("new_x", "qp_status", "admm_iters", "polish"):
        assert np.array_equal(cta[k], warp[k]), (k, np.abs(np.asarray(cta[k], float) - warp[k]).max())


@pytest.mark.parametrize("name", list(DESC))
def test_sqp_solve_factor_paths_identical(monkeypatch, name):
    d = DESC[name]()
    cta, warp = _both(monkeypatch, d, lambda p: p.solve())
    for k in ("x", "status", "n_qp_solves", "n_admm_iters"):
        assert np.array_equal(cta[k], warp[k]), (k, np.abs(np.asarray(cta[k], float) - warp[k]).max())
