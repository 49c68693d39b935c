"""The avoid_singularity term (AvoidSingularityTermInfo, kinematic_terms.cpp:586-642): hatching and its refusals, the
oracle's term (one-sided Jacobi SVD, err, forward-difference gradient) against numpy, and on the GPU (-m gpu) the
device's rows, QP and SQP against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from trajopt_b200 import api, capi, json_io, problems, robots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


def with_terms(d, extra, init=None, first=False):
    """d with `extra` appended to its terms (first: put before them)."""
    terms = list(extra) + list(d.terms) if first else list(d.terms) + list(extra)
    return capi.ProblemDesc(d.robot_spec, d.T, terms, d.init_traj if init is None else init,
                            fixed_timesteps=list(d._fixed_t), fixed_dofs=list(d._fixed_d), cart_targets=d.cart_targets,
                            obstacles=d.obstacles, sqp=d.c.sqp, qp=d.c.qp)


def cfg2_sing(role, B=8, T=12, coeff=1.0, lam=0.1, first=False):
    d = problems.config2(B=B, T=T)
    tool = d.robot_spec["tool"]
    return with_terms(d, [problems.avoid_singularity_term(role, 0, T - 1, tool, coeff, lam)], first=first)


# ---------------------------------------------------------------------------------------------------------------- CPU
def _planted(rng, D, smin):
    """a 6 x D matrix with singular values spread from 1 down to smin"""
    k = min(6, D)
    U, _ = np.linalg.qr(rng.standard_normal((6, k)))
    V, _ = np.linalg.qr(rng.standard_normal((D, k)))
    s = np.geomspace(1.0, smin, k) if k > 1 else np.array([smin])
    return U @ np.diag(s) @ V.T


@pytest.mark.parametrize("D", [2, 3, 6, 7, 14, 16])
def test_svd_matches_numpy(oracle, D):
    rng = np.random.default_rng(100 + D)
    cases = [rng.standard_normal((6, D))]
    cases += [_planted(rng, D, s) for s in (1e-8, 1e-6, 1e-3, 1e-1, 1.0)]
    z = rng.standard_normal((6, D))
    z[:, ::2] = 0.0  # zero columns (the dual arm: joints that do not move the link)
    cases.append(z)
    if D >= 2:  # exactly rank deficient: two equal columns
        r = rng.standard_normal((6, D))
        r[:, 1] = r[:, 0]
        cases.append(r)
    for J in cases:
        s, u, v = oracle.sing_svd_min(J)
        ref = np.linalg.svd(J, compute_uv=False)[-1]
        scale = np.linalg.norm(J, 2)
        if ref > 1e-10 * scale:
            assert abs(s - ref) <= 1e-12 * max(ref, 1e-4 * scale) + 1e-15 * scale, (s, ref)
            assert np.linalg.norm(J @ v - s * u) <= 1e-12 * scale
            assert np.linalg.norm(J.T @ u - s * v) <= 1e-12 * scale
        else:
            assert s <= 1e-12 * scale, (s, ref)


def _numpy_err_grad(robot, q, link, lam):
    J0 = robots.jacobian_numpy(robot, q, link)
    U, S, Vt = np.linalg.svd(J0, full_matrices=False)
    s, u, v = S[-1], U[:, -1], Vt[-1]
    err = 1.0 / (s + lam) - 1.0 / (0.1 + lam)
    g = np.zeros(q.size)
    for j in range(q.size):
        qk = q.copy()
        qk[j] += 1e-6
        g[j] = u @ ((robots.jacobian_numpy(robot, qk, link) - J0) / 1e-6) @ v
    return s, err, g * (-1.0 / (s + lam) ** 2)


@pytest.mark.parametrize("arm", ["pr2", "dual_right", "dual_left"])
def test_err_and_gradient_on_the_arms(oracle, arm):
    if arm == "pr2":
        d, link = problems.config2(B=2, T=6), None
    else:
        d, link = problems.config4(B=2, T=6), None
    robot = d.robot_spec
    link = robot["tool_left"] if arm == "dual_left" else robot["tool"]
    rng = np.random.default_rng(5)
    lo, hi = np.array(robot["lower"]), np.array(robot["upper"])
    for _ in range(6):
        q = rng.uniform(np.maximum(lo, -3), np.minimum(hi, 3))
        for lam in (0.1, 0.02):
            J, s, e, g = oracle.sing_err_grad(d, q, link, lam)
            np.testing.assert_allclose(J, robots.jacobian_numpy(robot, q, link), atol=1e-12)
            s_ref, e_ref, g_ref = _numpy_err_grad(robot, q, link, lam)
            assert abs(s - s_ref) <= 1e-12 * max(1.0, s_ref)
            assert abs(e - e_ref) <= 1e-10 * max(1.0, abs(e_ref))
            np.testing.assert_allclose(g, g_ref, atol=1e-7 * max(1.0, np.abs(g_ref).max()))
            # a central difference of err (sigma is simple at a random state)
            gc = np.zeros_like(q)
            for j in range(q.size):
                h = np.zeros_like(q)
                h[j] = 1e-5
                gc[j] = (oracle.sing_err_grad(d, q + h, link, lam)[2] - oracle.sing_err_grad(d, q - h, link, lam)[2]) / 2e-5
            np.testing.assert_allclose(g, gc, atol=1e-4 * max(1.0, np.abs(gc).max()))


def _create(desc):
    lib = capi.load_library()
    h = C.c_void_p()
    rc = lib.tb200_problem_create(C.byref(desc.c), 0, C.byref(h))
    msg = lib.tb200_last_error().decode()
    if rc == 0:
        lib.tb200_problem_destroy(h)
    return rc, msg


@pytest.mark.parametrize("kw,text", [
    (dict(link=99), "avoid_singularity link out of range"),
    (dict(link=-1), "avoid_singularity link out of range"),
    (dict(first=-1, last=-1), "avoid_singularity steps outside the trajectory"),
    (dict(first=0, last=12), "avoid_singularity steps outside the trajectory"),
    (dict(first=5, last=4), "avoid_singularity steps outside the trajectory"),
    (dict(lam=-0.1), "avoid_singularity lambda must be finite and >= 0"),
    (dict(lam=float("nan")), "avoid_singularity lambda must be finite and >= 0"),
    (dict(lam=float("inf")), "avoid_singularity lambda must be finite and >= 0"),
])
def test_description_errors(kw, text):
    d = problems.config2(B=2, T=12)
    a = dict(first=0, last=11, link=d.robot_spec["tool"], lam=0.1)
    a.update(kw)
    t = problems.avoid_singularity_term(capi.ROLE_CNT, a["first"], a["last"], a["link"], 1.0, a["lam"])
    rc, msg = _create(with_terms(d, [t]))
    assert rc == capi.ERR_INVALID and msg == text, (rc, msg)


def test_good_description_needs_a_device():
    import torch
    rc, msg = _create(cfg2_sing(capi.ROLE_CNT))
    assert rc == (0 if torch.cuda.is_available() else capi.ERR_NO_DEVICE), msg


def test_json_still_refused():
    doc = {"basic_info": {"n_steps": 4, "manip": "right_arm"},
           "costs": [{"type": "avoid_singularity", "params": {"link": "r_gripper_tool_frame"}}],
           "constraints": [], "init_info": {"type": "stationary"}}
    with pytest.raises(ValueError, match="failed to construct cost named avoid_singularity"):
        json_io.from_json(doc, robots.pr2_arm("r"), np.zeros((1, 7)))


def _layout(oracle, d):
    L = oracle.layout(d)
    return L.n_costs, L.n_cnts, L.n_cart_rows, L.cart_jac_stride


def test_model_hatching(oracle):
    """object counts and places: costs after the other costs, constraints after every EQ and INEQ constraint; with the
    term first, its objects and cart rows come first in their lists"""
    base = _layout(oracle, problems.config2(B=2, T=12))
    for role in (capi.ROLE_COST, capi.ROLE_CNT):
        nc, nk, R, CS = _layout(oracle, cfg2_sing(role, B=2))
        assert (nc - base[0], nk - base[1]) == ((12, 0) if role == capi.ROLE_COST else (0, 12))
        assert R == base[2] + 12 and CS == base[3]
        last, first = cfg2_sing(role, B=2), cfg2_sing(role, B=2, first=True)
        assert _layout(oracle, first) == (nc, nk, R, CS)
        tl, sl = oracle.objects(last)
        tf, sf = oracle.objects(first)
        at = np.arange(12) + (base[0] if role == capi.ROLE_COST else nc + base[1])
        assert (tl[at] == len(last.terms) - 1).all() and (sl[at] == np.arange(12)).all()
        assert (tf == 0).sum() == 12 and (sf[tf == 0] == np.arange(12)).all()
        x = last.init_traj + 0.01
        cl, cf = oracle.convexify_batch(last, x), oracle.convexify_batch(first, x)
        assert cf["cart_err"][:, :12].tobytes() == cl["cart_err"][:, -12:].tobytes()
        assert cf["cart_err"][:, 12:].tobytes() == cl["cart_err"][:, :-12].tobytes()
        assert sorted(cf["cost_vals"].ravel().tolist() + cf["cnt_viols"].ravel().tolist()) == \
            sorted(cl["cost_vals"].ravel().tolist() + cl["cnt_viols"].ravel().tolist())


def _near_singular(B=64, T=12, seed=3):
    """PR2 arm moving through elbow flex = 0 (its upper limit), where the upper arm and forearm axes line up: sigma of
    the tool Jacobian dips towards 0 on the way."""
    robot = robots.pr2_arm("r", with_spheres=False)
    rng = np.random.default_rng(seed)
    q0 = np.array([-0.5, 0.3, -1.0, -1.2, 0.5, -0.6, 0.2])
    q1 = np.array([-0.3, 0.5, -0.8, -0.0005, 0.7, -0.05, 0.4])
    q0s = q0 + 0.02 * rng.standard_normal((B, 7))
    q1s = q1 + 0.02 * rng.standard_normal((B, 7))
    q1s[:, 3] = np.minimum(q1s[:, 3], -1e-3)
    q1s[:, 5] = np.minimum(q1s[:, 5], -1e-3)
    init = problems.interpolate(q0s, q1s, T)
    terms = [problems.joint_term(capi.TERM_JOINT_VEL, capi.ROLE_COST, 7, 0, T - 1),
             problems.joint_term(capi.TERM_JOINT_POS, capi.ROLE_CNT, 7, T - 1, T - 1, targets=q1)]
    return robot, capi.ProblemDesc(robot, T, terms, init, fixed_timesteps=[0])


def test_behaviour_on_the_model(oracle):
    robot, d = _near_singular(B=4)
    tool = robot["tool"]
    sig = lambda x: np.array([[robots.smallest_singular_value(robot, x[b, t], tool) for t in range(d.T)]  # noqa: E731
                              for b in range(d.B)])
    base = oracle.solve_batch(d)
    s0 = sig(base["x"])
    assert (s0.min(axis=1) < 0.1).all()
    # (the goal itself is close to singular: the constraint covers the steps between start and goal)
    cnt = with_terms(d, [problems.avoid_singularity_term(capi.ROLE_CNT, 1, d.T - 2, tool)])
    got = oracle.solve_batch(cnt)
    s1 = sig(got["x"])
    assert (got["status"] == capi.OPT_CONVERGED).all(), got["status"]
    # violation <= cnt_tolerance: 1/(s + 0.1) - 5 <= 1e-4
    assert (1.0 / (s1[:, 1:-1] + 0.1) - 5.0 <= 1.1e-4).all(), s1.min()
    cost = with_terms(d, [problems.avoid_singularity_term(capi.ROLE_COST, 1, d.T - 1, tool)])
    init_cost = oracle.convexify_batch(cost, cost.init_traj)["cost_vals"][:, -(d.T - 1):].sum(axis=1)
    got_c = oracle.solve_batch(cost)
    end_cost = got_c["cost_vals"][:, -(d.T - 1):].sum(axis=1)
    assert (end_cost < init_cost).all()
    # the quirk: the ABS cost is smallest at sigma = 0.1, so sigma far above 0.1 is pulled down as well
    sc = sig(got_c["x"])[:, 1:]
    si = sig(cost.init_traj)[:, 1:]
    assert np.abs(sc - 0.1).mean() < np.abs(si - 0.1).mean()


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cases():
    d3 = problems.config3(B=4, T=12)
    d4 = problems.config4(B=4, T=12)
    out = {}
    for role, rn in ((capi.ROLE_COST, "cost"), (capi.ROLE_CNT, "cnt")):
        out[f"cfg2_{rn}"] = cfg2_sing(role, B=4, coeff=2.0, lam=0.05)
        out[f"cfg3_{rn}"] = with_terms(d3, [problems.avoid_singularity_term(role, 1, 11, d3.robot_spec["tool"], 1.5)])
        out[f"cfg4_{rn}"] = with_terms(d4, [
            problems.avoid_singularity_term(role, 0, 11, d4.robot_spec["tool"]),
            problems.avoid_singularity_term(role, 2, 9, d4.robot_spec["tool_left"], 0.5, 0.2)])
    out["cfg2_cnt_first"] = cfg2_sing(capi.ROLE_CNT, B=4, coeff=2.0, lam=0.05, first=True)
    return out


_CASES = {}


def _case(name):
    if not _CASES:
        _CASES.update(_cases())
    return _CASES[name]


_NAMES = ["cfg2_cost", "cfg2_cnt", "cfg3_cost", "cfg3_cnt", "cfg4_cost", "cfg4_cnt"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", _NAMES)
def test_convexify_rows_match_model(oracle, name):
    d = _case(name)
    rng = np.random.default_rng(11)
    x = d.init_traj + 0.05 * rng.standard_normal(d.init_traj.shape)
    p = api.Problem(d)
    got = p.convexify(x)
    term, step = p.objects()
    p.close()
    ref = oracle.convexify_batch(d, x)
    nr = ref["cart_err"].shape[1]
    n_sing = sum(t.last_step - t.first_step + 1 for t in d.terms if t.kind == capi.TERM_AVOID_SINGULARITY)
    sl = slice(nr - n_sing, nr)
    np.testing.assert_allclose(got["cart_err"][:, sl], ref["cart_err"][:, sl], rtol=1e-10, atol=1e-13)
    c = max(abs(t.coeffs[0]) for t in d.terms if t.kind == capi.TERM_AVOID_SINGULARITY)
    np.testing.assert_allclose(got["cart_jac"][:, sl], ref["cart_jac"][:, sl], rtol=0, atol=1e-7 * c)
    np.testing.assert_allclose(got["cart_err"][:, :nr - n_sing], ref["cart_err"][:, :nr - n_sing], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(got["cost_vals"], ref["cost_vals"], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(got["cnt_viols"], ref["cnt_viols"], rtol=1e-9, atol=1e-12)
    # the objects name their term and step: the avoid_singularity objects one per step, last in their list
    k_sing = [k for k, t in enumerate(d.terms) if t.kind == capi.TERM_AVOID_SINGULARITY]
    want = [(k, s) for k in k_sing for s in range(d.terms[k].first_step, d.terms[k].last_step + 1)]
    is_cnt = d.terms[k_sing[0]].role == capi.ROLE_CNT
    nc = got["cost_vals"].shape[1]
    pairs = list(zip(term.tolist(), step.tolist()))
    assert (pairs[len(pairs) - len(want):] if is_cnt else pairs[nc - len(want):nc]) == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", _NAMES)
@pytest.mark.parametrize("trust", [0.1, 0.01])
def test_qp_solve_matches_model(oracle, name, trust):
    d = _case(name)
    x = d.init_traj.copy()
    p = api.Problem(d)
    got = p.qp_solve(x, trust, 10.0)
    p.close()
    ref = oracle.qp_solve_batch(d, x, trust, 10.0)
    assert (got["qp_status"] == ref["qp_status"]).all()
    np.testing.assert_allclose(got["new_x"], ref["new_x"], atol=1e-5)
    np.testing.assert_allclose(got["model_cnt_viols"], ref["model_cnt_viols"], atol=1e-6)
    np.testing.assert_allclose(got["model_cost_vals"], ref["model_cost_vals"], rtol=1e-6, atol=1e-7)


def _compare_sqp(got, ref):
    assert (got["status"] == ref["status"]).all(), (got["status"], ref["status"])
    assert (got["n_qp_solves"] == ref["n_qp_solves"]).all(), (got["n_qp_solves"], ref["n_qp_solves"])
    np.testing.assert_allclose(got["total_cost"], ref["total_cost"], atol=1e-6)


@pytest.mark.gpu
def test_sqp_near_singular_batch_matches_model(oracle):
    robot, d = _near_singular(B=64)
    cnt = with_terms(d, [problems.avoid_singularity_term(capi.ROLE_CNT, 1, d.T - 2, robot["tool"])])
    got = api.solve(cnt)
    ref = oracle.solve_batch(cnt)
    _compare_sqp(got, ref)
    s = np.array([[robots.smallest_singular_value(robot, got["x"][b, t], robot["tool"]) for t in range(1, d.T - 1)]
                  for b in range(d.B)])
    ok = got["status"] == capi.OPT_CONVERGED
    assert ok.any() and (1.0 / (s[ok] + 0.1) - 5.0 <= 1.1e-4).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2_cost", "cfg2_cnt", "cfg4_cost", "cfg2_cnt_first"])
def test_sqp_matches_model(oracle, name):
    d = _case(name)
    _compare_sqp(api.solve(d), oracle.solve_batch(d))


def _solve_with_trace(d, cap=600):
    """GPU solve with the decision trace on, and per trajectory whether any of its QPs ended WITHOUT a KKT-verified polished
    point (iteration limit, or a polish rejected / accepted unverified): such a QP returns an ADMM iterate that is only
    eps-accurate, so that trajectory cannot be compared step by step (DESIGN.md deviation D2; test_gpu_parity.py)."""
    p = api.Problem(d)
    p.lib.tb200_debug_enable_trace(p.handle, cap)
    got = p.solve()
    tr = np.zeros((d.B, cap, 14))
    tl = np.zeros(d.B, np.int32)
    p.lib.tb200_debug_fetch_trace(p.handle, tr.ctypes.data_as(_dbl_p), tl.ctypes.data_as(_i32_p))
    p.close()
    hit = np.array([(tr[b, :tl[b], 7] >= d.c.qp.max_iter).any() or (tr[b, :tl[b], 12] != 1).any() for b in range(d.B)])
    return got, hit


def configs2_every_step(B=256):
    d = problems.config2(B=B)
    return with_terms(d, [problems.avoid_singularity_term(capi.ROLE_COST, 0, d.T - 1, d.robot_spec["tool"])])


@pytest.mark.gpu
def test_sqp_configs2_every_step_batch_256(oracle):
    """configs[2] with the cost on every step, all 256 trajectories, with the rule of test_gpu_parity.py: a trajectory
    with a QP that ended without a KKT-verified polished point is not compared step by step (at least 3 of 4 must be
    comparable); every other one has the model's status and QP count, and its final cost within 1e-4 relative.  (The
    forward-difference gradient turns last-bit differences of the two FKs into ~1e-9 in the rows; over ~50 QPs that moves
    the final cost of a few trajectories by more than 1e-6: on an H100, 6 of 236 comparable trajectories, at most
    2.8e-4 absolute and 4.8e-5 relative.)"""
    d = configs2_every_step()
    got, hit = _solve_with_trace(d)
    ref = oracle.solve_batch(d)
    ok = ~hit
    assert ok.mean() >= 0.75, np.nonzero(hit)[0]
    assert (got["status"][ok] == ref["status"][ok]).all(), np.nonzero(ok & (got["status"] != ref["status"]))[0]
    assert (got["n_qp_solves"][ok] == ref["n_qp_solves"][ok]).all(), \
        np.nonzero(ok & (got["n_qp_solves"] != ref["n_qp_solves"]))[0]
    np.testing.assert_allclose(got["total_cost"][ok], ref["total_cost"][ok], rtol=1e-4, atol=1e-6)
    assert (got["status"] != capi.OPT_INVALID).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2_cost", "cfg2_cnt", "cfg4_cnt"])
def test_sqp_log_matches_the_model(oracle, name):
    """The SQP log with the term against the model's driver: per record the decision (round, iteration, action), QP
    failures, trust box to 1e-8 and merits to 1e-7 (test_sqp_log.py holds the oracle to 1e-8; the forward-difference
    rows of the term move a merit of ~100 by ~1e-6); the objects name their term and step where the model puts them."""
    d = _case(name)
    p = api.Problem(d)
    p.set_sqp_log(512)
    got = p.solve()
    L = p.sqp_log()
    term, step = p.objects()
    nc = p.layout.n_costs
    p.close()
    ref = oracle.solve_batch(d, records=512)
    _compare_sqp(got, ref)
    want_term, want_step = oracle.objects(d)
    assert len(want_term) == nc + len(got["cnt_viols"][0])
    np.testing.assert_array_equal(term, want_term)
    np.testing.assert_array_equal(step, want_step)
    for b in range(d.B):
        n = L["n_records"][b] - 1
        assert n == got["n_qp_solves"][b] and n == ref["log"]["n_records"][b] - 1, b
        tr = ref["log"]["trace"][b, 1:n + 1]
        sl = slice(1, n + 1)
        dev = np.stack([L["merit_round"][b, sl], L["iter"][b, sl], L["action"][b, sl]], 1)
        np.testing.assert_array_equal(dev, tr[:, [0, 1, 8]])
        np.testing.assert_array_equal((L["qp_status"][b, sl] == 1) | (L["qp_status"][b, sl] == 2),
                                      (tr[:, 6] == 1) | (tr[:, 6] == 2))
        okr = L["action"][b, sl] != 3
        np.testing.assert_allclose(L["trust_box_size"][b, sl], tr[:, 2], rtol=1e-8, atol=1e-8)
        for c, k in ((3, "old_merit"), (4, "model_merit"), (5, "new_merit")):
            np.testing.assert_allclose(L[k][b, sl][okr], tr[okr, c], rtol=1e-7, atol=1e-8)


@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    capi.load_library()  # the CUDA build must exist (no GPU needed to load it)
    csrc = os.path.join(ROOT, "trajopt_b200", "csrc")
    out = str(tmp_path_factory.mktemp("ash") / "avoid_singularity_host")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "avoid_singularity_host.cpp"), "-o", out, "-L", csrc, "-ltrajopt_b200",
           "-Wl,-rpath," + csrc, "-Wl,--allow-shlib-undefined"]
    subprocess.run(cmd, check=True)
    return out


@pytest.mark.parametrize("mode,rc,text", [
    ("ok", 0, "kind 6 role 1 link 2 first 1 last 4 coeff 2.5 lambda 0.050000000000000003"),
    ("cnt", 0, "kind 6 role 2 link 2 first 1 last 4 coeff 1 lambda 0.10000000000000001"),
    ("two_coeffs", 3, "runtime_error: avoid_singularity: coeffs has more than one element"),
    ("unknown_link", 3, 'runtime_error: link "nowhere" is not part of the manipulator model'),
    ("default_steps", 3, "runtime_error: avoid_singularity: steps outside the trajectory"),
    ("past_the_end", 3, "runtime_error: avoid_singularity: steps outside the trajectory"),
    ("reversed", 3, "runtime_error: avoid_singularity: steps outside the trajectory"),
])
def test_cpp_layer_hatch(host_bin, mode, rc, text):
    """AvoidSingularityTermInfo::hatch: the term it writes (empty coeffs: 1; lambda's default 0.1) and its three refusals"""
    r = subprocess.run([host_bin, mode], capture_output=True, text=True)
    assert (r.returncode, r.stdout.strip()) == (rc, text)
