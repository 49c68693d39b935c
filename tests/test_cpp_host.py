"""The C++ host layer (include/trajopt_b200.hpp: ProblemConstructionInfo / TermInfo / ConstructProblem /
OptimizeProblem under the reference's names) against the Python mirror of the same C ABI.
CPU: it compiles, flattens configs[2] to the byte-identical POD description, and fails loudly without a device.
GPU (-m gpu): solving through it gives the results of the Python path."""
import subprocess

import numpy as np
import pytest

import cpp_host
from trajopt_b200 import api, capi, problems, robots  # noqa: F401


@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "host_mirror")


def _case(tmp_path):
    d = problems.config2(B=3, T=10)
    return d, cpp_host.write_problem(tmp_path / "in.txt", d)


def test_cpp_host_flattens_to_the_same_description(host_bin, tmp_path):
    """configs[2] as tests/cpp/host_input.hpp writes it, for every host program that solves it."""
    d, path = _case(tmp_path)
    out = subprocess.run([host_bin, path, "dump"], check=True, capture_output=True, text=True).stdout.splitlines()
    assert out[0] == f"n_terms {len(d.terms)} n_cart_targets 1 n_fixed 1"
    assert out[1].split()[1] == bytes(d._terms).hex()  # tb200_term[] byte for byte
    init = np.array(out[2].split()[1:], float).reshape(d.init_traj.shape)
    np.testing.assert_allclose(init, d.init_traj, rtol=0, atol=1e-14)  # LinSpaced vs numpy linspace rounding
    tg = np.array(out[3].split()[1:], float).reshape(d.cart_targets.shape)
    np.testing.assert_array_equal(tg, d.cart_targets)


def test_cpp_host_fails_loudly_without_a_device(host_bin, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    _, path = _case(tmp_path)
    r = subprocess.run([host_bin, path, "solve"], capture_output=True, text=True)
    assert r.returncode == 3 and "no CUDA device" in r.stderr  # std::runtime_error, never a CPU fallback


JSON_DOC = """
{
  "basic_info": {"n_steps": 10, "manip": "right_arm", "fixed_timesteps": [0], "convex_solver": "OSQP"},
  "opt_info": {"max_iter": 40, "trust_box_size": 0.2},
  "costs": [
    {"type": "joint_vel", "params": {"coeffs": [2], "targets": [0]}},
    {"type": "joint_acc", "name": "smooth", "params": {"targets": [0, 0, 0, 0, 0, 0, 0], "upper_tols": [0.1], "lower_tols": [-0.1]}},
    {"type": "collision", "params": {"coeffs": 20, "dist_pen": 0.025, "evaluator_type": 4, "fixed_steps": [0],
                                      "longest_valid_segment_length": 0.05}}
  ],
  "constraints": [
    {"type": "cart_pose", "params": {"timestep": 9, "source_frame": "link9", "target_frame": "base_footprint",
                                      "target_frame_offset_xyz": [0.6, -0.2, 0.9], "target_frame_offset_wxyz": [0, 0, 1, 0],
                                      "rot_coeffs": [1, 1, 0]}},
    {"type": "cart_vel", "params": {"first_step": 0, "last_step": 8, "max_displacement": 0.05, "link": "link9"}},
    {"type": "joint_pos", "name": "end", "params": {"targets": [0.1, 0.2, 0.3, -0.4, 0.5, -0.6, 0.7], "first_step": 9, "last_step": 9}}
  ],
  "init_info": {"type": "JOINT_interpolated", "endpoint": [0.1, 0.2, 0.3, -0.4, 0.5, -0.6, 0.7]}
}
"""


def test_json_front_end_matches_the_struct_description(host_bin, tmp_path):
    """ProblemConstructionInfo::fromJson in the reference's schema (SURVEY.md Appendix A) against the same description
    written with the Python mirror: byte-identical terms, same initial trajectory, opt_info overrides taken."""
    d, path = _case(tmp_path)
    jpath = str(tmp_path / "prob.json")
    open(jpath, "w").write(JSON_DOC)
    out = subprocess.run([host_bin, path, "json", jpath], check=True, capture_output=True, text=True).stdout.splitlines()
    T, D = 10, 7
    tool = d.robot_spec["tool"]
    assert tool == 9  # "link9" above
    terms = [problems.joint_term(capi.TERM_JOINT_VEL, capi.ROLE_COST, D, 0, T - 1, coeffs=2.0, T=T),
             problems.joint_term(capi.TERM_JOINT_ACC, capi.ROLE_COST, D, 0, T - 1, upper=0.1, lower=-0.1, T=T),
             problems.collision_term(capi.ROLE_COST, 0, T - 1, margin=0.025, coeff=20.0, buffer=0.5, fixed_steps=[0],
                                     evaluator=capi.COLL_LVS_CONTINUOUS, lvs=0.05),
             problems.cart_pose_term(capi.ROLE_CNT, 9, tool, target_slot=0, rot_coeffs=(1, 1, 0)),
             problems.cart_vel_term(capi.ROLE_CNT, 0, 8, tool, 0.05),
             problems.joint_term(capi.TERM_JOINT_POS, capi.ROLE_CNT, D, 9, 9, targets=[0.1, 0.2, 0.3, -0.4, 0.5, -0.6, 0.7], T=T)]
    ref_terms = (capi.Term * len(terms))(*terms)
    assert out[0] == "n_terms 6 n_cart_targets 1 n_fixed 1 max_iter 40 trust 0.20000000000000001"
    assert out[1].split()[1] == bytes(ref_terms).hex()
    init = np.array(out[2].split()[1:], float).reshape(d.B, T, D)
    q0 = d.init_traj[:, 0]
    want = problems.interpolate(q0, np.tile([0.1, 0.2, 0.3, -0.4, 0.5, -0.6, 0.7], (d.B, 1)), T)
    np.testing.assert_allclose(init, want, rtol=0, atol=1e-14)
    tg = np.array(out[3].split()[1:], float).reshape(d.B, 7)
    np.testing.assert_array_equal(tg, np.tile([0.6, -0.2, 0.9, 0, 0, 1, 0], (d.B, 1)))


def test_python_json_loader_is_the_twin_of_the_cpp_one(host_bin, tmp_path):
    from trajopt_b200 import json_io
    d, path = _case(tmp_path)
    jpath = str(tmp_path / "prob.json")
    open(jpath, "w").write(JSON_DOC)
    out = subprocess.run([host_bin, path, "json", jpath], check=True, capture_output=True, text=True).stdout.splitlines()
    pd = json_io.from_json(JSON_DOC, d.robot_spec, d.init_traj[:, 0], obstacles=d.obstacles)
    assert out[1].split()[1] == bytes(pd._terms).hex()
    np.testing.assert_allclose(np.array(out[2].split()[1:], float).reshape(pd.init_traj.shape), pd.init_traj, rtol=0, atol=1e-14)
    np.testing.assert_array_equal(np.array(out[3].split()[1:], float).reshape(pd.cart_targets.shape), pd.cart_targets)
    assert pd.c.sqp.max_iter == 40 and pd.c.sqp.trust_box_size == 0.2
    with pytest.raises(ValueError, match="illegal field"):
        json_io.from_json(JSON_DOC.replace('"targets": [0]}', '"targets": [0], "bogus": 1}'), d.robot_spec, d.init_traj[:, 0])


def test_python_json_loader_solves_on_the_oracle(oracle):
    """A document in the reference's schema end to end on the CPU path (arm_around_table.json's shape: joint_vel cost,
    collision cost with the LVS_CONTINUOUS evaluator and fixed end steps, joint_pos end constraint, given_traj init)."""
    from trajopt_b200 import json_io
    robot = robots.pr2_arm("r", with_spheres=True)
    q0 = np.array([-1.832, -0.332, -1.011, -1.437, -1.1, -1.926, 3.074])
    q1 = np.array([0.062, 1.287, 0.1, -1.554, -3.011, -0.268, 2.988])
    traj = [list(q0 + (q1 - q0) * k / 5) for k in range(6)]
    doc = {"basic_info": {"n_steps": 6, "manip": "right_arm", "fixed_timesteps": [0]},
           "costs": [{"type": "joint_vel", "params": {"coeffs": [1], "targets": [0] * 7}},
                     {"type": "collision", "params": {"coeffs": 20, "dist_pen": 0.025, "evaluator_type": 4, "fixed_steps": [0, 5],
                                                      "longest_valid_segment_length": 0.2}}],
           "constraints": [{"type": "joint_pos", "name": "joint0",
                            "params": {"coeffs": [1] * 7, "targets": list(q1), "first_step": 5, "last_step": 5}}],
           "init_info": {"type": "given_traj", "data": traj}}
    obstacles = np.array([[[0.9, 0.4, 1.6, 0.05]]])  # one small sphere away from the arm
    pd = json_io.from_json(doc, robot, q0[None], obstacles=obstacles)
    r = oracle.solve_batch(pd)
    assert r["status"][0] == capi.OPT_CONVERGED
    np.testing.assert_allclose(r["x"][0, 0], q0, atol=1e-9)       # fixed_timesteps
    np.testing.assert_allclose(r["x"][0, 5], q1, atol=1e-3)       # the joint_pos constraint


@pytest.mark.parametrize("bad,msg", [
    ('"params": {"coeffs": [2], "targets": [0], "bogus": 1}', "illegal field"),   # ensure_only_members
    ('"params": {"coeffs": [2]}', "missing field: targets")])
def test_json_front_end_rejects_what_the_reference_rejects(host_bin, tmp_path, bad, msg):
    _, path = _case(tmp_path)
    jpath = str(tmp_path / "bad.json")
    open(jpath, "w").write(JSON_DOC.replace('"params": {"coeffs": [2], "targets": [0]}', bad))
    r = subprocess.run([host_bin, path, "json", jpath], capture_output=True, text=True)
    assert r.returncode == 3 and msg in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["solve", "solve_ref"])
def test_cpp_host_solves_like_the_python_path(host_bin, tmp_path, mode):
    """OptimizeWithParams runs with pci.opt_info; OptimizeProblem reproduces the reference's hard-coded overrides
    (max_iter 40, min_approx_improve_frac 1e-3, improve_ratio_threshold 0.2, initial_merit_error_coeff 20 on top of the
    optimizer defaults, problem_description.cpp:394-408)."""
    d, path = _case(tmp_path)
    out = subprocess.run([host_bin, path, mode], check=True, capture_output=True, text=True).stdout.splitlines()
    if mode == "solve_ref":
        d.c.sqp = capi.default_sqp_params()
        d.c.sqp.max_iter, d.c.sqp.min_approx_improve_frac = 40, 1e-3
        d.c.sqp.improve_ratio_threshold, d.c.sqp.initial_merit_error_coeff = 0.2, 20.0
    ref = api.solve(d)
    assert len(out) == d.B
    for b, line in enumerate(out):
        v = line.split()
        assert int(v[1]) == ref["status"][b] and int(v[3]) == ref["n_qp_solves"][b]
        assert abs(float(v[2]) - ref["total_cost"][b]) < 1e-6
        np.testing.assert_allclose(np.array(v[5:], float), ref["x"][b].ravel(), atol=1e-5)
