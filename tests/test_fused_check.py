"""The termination check fused into the partition-inverse ADMM block and the polish passes of polish_passes (short
trajectories) against the generic passes
(TB200_GENERIC_QP_PASSES=1, read when a problem is created): same decisions, same solutions.  -m gpu."""
import numpy as np
import pytest

from trajopt_b200 import api, problems

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("cfg", ["cfg1", "cfg2"])
@pytest.mark.parametrize("trust", [0.1, 0.01])
def test_qp_solve_fused_check_matches_generic(monkeypatch, cfg, trust):
    d = getattr(problems, {"cfg1": "config1", "cfg2": "config2"}[cfg])(B=32, T=30)
    x = d.init_traj.copy()
    gen, fus = _both(monkeypatch, d, lambda p: p.qp_solve(x, trust, 10.0))
    assert (gen["qp_status"] == fus["qp_status"]).all()
    assert (gen["admm_iters"] == fus["admm_iters"]).all(), (gen["admm_iters"], fus["admm_iters"])
    assert (gen["polish"] == fus["polish"]).all()
    np.testing.assert_allclose(fus["new_x"], gen["new_x"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("cfg", ["cfg1", "cfg2"])
def test_sqp_solve_fused_check_matches_generic(monkeypatch, cfg):
    d = getattr(problems, {"cfg1": "config1", "cfg2": "config2"}[cfg])(B=32, T=30)
    gen, fus = _both(monkeypatch, d, lambda p: p.solve())
    for k in ("status", "n_qp_solves", "n_admm_iters"):
        assert (gen[k] == fus[k]).all(), (k, gen[k], fus[k])
    np.testing.assert_allclose(fus["x"], gen["x"], rtol=0, atol=1e-9)
