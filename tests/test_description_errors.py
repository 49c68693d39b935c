"""tb200_problem_create checks and flattens the description before it touches a device: a bad or unsupported
description gets the reference's kind of answer (an error code + message, PRINT_AND_THROW in the reference) on any
machine, and a good one ends in TB200_ERR_NO_DEVICE here (no GPU, no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

from trajopt_b200 import capi, problems


def _create(desc):
    lib = capi.load_library()
    h = C.c_void_p()
    rc = lib.tb200_problem_create(C.byref(desc.c), 0, C.byref(h))
    msg = lib.tb200_last_error().decode()
    if rc == 0:
        lib.tb200_problem_destroy(h)
    return rc, msg


def _no_device():
    import torch
    return not torch.cuda.is_available()


def test_good_description_needs_a_device():
    rc, msg = _create(problems.config2(B=2, T=10))
    if _no_device():
        assert rc == capi.ERR_NO_DEVICE and "no CPU fallback" in msg
    else:
        assert rc == 0


def _variant(edit, maker=lambda: problems.config2(B=2, T=10)):
    d = maker()
    edit(d)
    return _create(d)


def _set_term(d, k, **kw):
    for name, v in kw.items():
        setattr(d._terms[k], name, v)


def _moving_segment(d):
    return next(s for s in d._segs if s.joint_type != capi.JOINT_FIXED)


def _nine_joint_objects():
    d = problems.config2(B=2, T=10)
    extra = [problems.joint_term(capi.TERM_JOINT_VEL, capi.ROLE_COST, d.D, 0, d.T - 1) for _ in range(7)]
    return capi.ProblemDesc(d.robot_spec, d.T, d.terms + extra, d.init_traj, fixed_timesteps=[0],
                            cart_targets=d.cart_targets, obstacles=d.obstacles)


@pytest.mark.parametrize("edit,code,text", [
    (lambda d: setattr(d.c, "n_steps", 0), capi.ERR_INVALID, "n_steps out of range"),
    (lambda d: setattr(d.c, "batch", 0), capi.ERR_INVALID, "batch must be >= 1"),
    (lambda d: _set_term(d, 2, link=99), capi.ERR_INVALID, "cart_pose link out of range"),
    (lambda d: _set_term(d, 2, first_step=77), capi.ERR_INVALID, "cart_pose timestep outside the trajectory"),
    (lambda d: _set_term(d, 3, evaluator_type=capi.COLL_LVS_DISCRETE, longest_valid_segment_length=0.0), capi.ERR_INVALID,
     "longest_valid_segment_length must be positive"),
    (lambda d: _set_term(d, 3, evaluator_type=9), capi.ERR_INVALID, "unknown collision evaluator type"),
    (lambda d: _set_term(d, 0, role=7), capi.ERR_INVALID, "term role must be COST or CNT"),
    (lambda d: _set_term(d, 0, kind=42), capi.ERR_INVALID, "unknown term kind"),
    (lambda d: _set_term(d, 0, last_step=500), capi.ERR_INVALID, "joint term steps outside the trajectory"),
    (lambda d: setattr(d._segs[1], "parent", 1), capi.ERR_INVALID, "segments must be topologically ordered"),
    (lambda d: setattr(_moving_segment(d), "q_index", 99), capi.ERR_INVALID, "bad q_index"),
    (lambda d: setattr(d._spheres[0], "segment", 999), capi.ERR_INVALID, "sphere attached to a bad segment"),
    (lambda d: setattr(d.c.robot, "n_segments", 0), capi.ERR_INVALID, "n_segments out of range"),
    (lambda d: setattr(d.c.robot, "n_spheres", 33), capi.ERR_INVALID, "too many collision spheres"),
    (lambda d: setattr(d.c, "n_obstacles", 0), capi.ERR_INVALID, "collision term needs robot spheres and obstacles"),
    (lambda d: _set_term(d, 3, last_step=50), capi.ERR_INVALID, "collision step outside the trajectory"),
    (lambda d: _set_term(d, 2, kind=capi.TERM_CART_VEL, link=99), capi.ERR_INVALID, "cart_vel link out of range"),
    (lambda d: _set_term(d, 2, kind=capi.TERM_CART_VEL, first_step=0, last_step=9), capi.ERR_INVALID,
     "cart_vel: step pair beyond the trajectory"),
    (lambda d: _set_term(d, 2, target_slot=1), capi.ERR_INVALID, "cart_pose target_slot out of range"),
    (lambda d: _set_term(d, 1, first_step=5, last_step=6), capi.ERR_INVALID, "joint term: trajectory is too short"),
])
def test_bad_descriptions_are_refused_before_the_device(edit, code, text):
    rc, msg = _variant(edit)
    assert rc == code and text in msg, (rc, msg)


def test_fixed_dof_outside_the_robot():
    d = problems.config_variants(B=1, T=10)
    d._fixed_d[0] = 7
    rc, msg = _create(d)
    assert rc == capi.ERR_INVALID and "DOF(aka Joint) indice is greater than the number of DOF available." in msg


def test_more_than_eight_joint_objects_are_refused():
    rc, msg = _create(_nine_joint_objects())
    assert rc == capi.ERR_UNSUPPORTED and "more than 8 joint-space cost/constraint objects" in msg, (rc, msg)


@pytest.mark.parametrize("edit,text", [
    # the robot is checked before the terms, the terms before the fixed timesteps
    (lambda d: (setattr(d._spheres[0], "segment", 999), _set_term(d, 3, evaluator_type=9)), "sphere attached to a bad segment"),
    (lambda d: (d._fixed_t.__setitem__(0, 10), _set_term(d, 0, role=7)), "term role must be COST or CNT"),
])
def test_the_first_fault_is_reported(edit, text):
    rc, msg = _variant(edit)
    assert rc == capi.ERR_INVALID and text in msg, (rc, msg)


def test_fixed_timestep_outside_the_trajectory():
    d = problems.config1(B=1, T=10)
    d._fixed_t[0] = 10
    rc, msg = _create(d)
    assert rc == capi.ERR_INVALID and "Fixed timestep index is outside the bounds" in msg  # the reference's text


def test_full_size_configs_pass_validation():
    """configs[3] at its full length (50 waypoints: 25 factor blocks) and the 14-DOF dual arm of configs[4] (factor
    blocks of 28, kept in global memory) are accepted: validation ends at the device check."""
    from trajopt_b200 import robots
    ok = capi.ERR_NO_DEVICE if _no_device() else 0
    rc, msg = _create(problems.config3(B=1, T=50))
    assert rc == ok, (rc, msg)
    robot = robots.pr2_dual_arm()
    d = capi.ProblemDesc(robot, 10, [problems.joint_term(capi.TERM_JOINT_VEL, capi.ROLE_COST, 14, 0, 9)], np.zeros((1, 10, 14)))
    rc, msg = _create(d)
    assert rc == ok, (rc, msg)


def test_non_positive_lvs_is_refused():
    rc, msg = _create(problems.config3(B=1, T=12, via_every=4, lvs=0.0))
    assert rc == capi.ERR_INVALID and "longest_valid_segment_length" in msg, (rc, msg)


def test_null_arrays_with_positive_counts_are_refused():
    d = problems.config2(B=1, T=10)
    d.c.obstacles = None
    rc, msg = _create(d)
    assert rc == capi.ERR_INVALID and "obstacles is NULL" in msg, (rc, msg)
    d = problems.config2(B=1, T=10)
    d.c.cart_targets = None
    rc, msg = _create(d)
    assert rc == capi.ERR_INVALID and "cart_targets is NULL" in msg, (rc, msg)
    d = problems.config2(B=1, T=10)
    _set_term(d, 3, n_fixed_steps=9)
    rc, msg = _create(d)
    assert rc == capi.ERR_INVALID and "n_fixed_steps" in msg, (rc, msg)


def test_mixing_discrete_and_continuous_collision_is_refused():
    d = problems.config2(B=1, T=10)
    terms = list(d.terms) + [problems.collision_term(capi.ROLE_COST, 0, 9, 0.02, 20.0, evaluator=capi.COLL_CONTINUOUS)]
    d2 = capi.ProblemDesc(d.robot_spec, 10, terms, d.init_traj, fixed_timesteps=[0], cart_targets=d.cart_targets, obstacles=d.obstacles)
    rc, msg = _create(d2)
    assert rc == capi.ERR_UNSUPPORTED and "discrete and continuous collision terms" in msg
