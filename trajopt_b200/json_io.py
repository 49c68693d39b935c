"""The reference's problem JSON (ProblemConstructionInfo::fromJson, trajopt/src/problem_description.cpp:118-308 and the
fromJson of each TermInfo; SURVEY.md Appendix A) -> ProblemDesc, for the terms of the device path.  Python twin of
include/trajopt_b200_json.hpp: same keys, defaults, single-value broadcast, unknown-key rejection and error texts.
One document describes one problem; it is repeated for `batch` problems that differ in their start state."""
import json

import numpy as np

from . import capi, problems

_JOINT_KINDS = {"joint_pos": capi.TERM_JOINT_POS, "joint_vel": capi.TERM_JOINT_VEL, "joint_acc": capi.TERM_JOINT_ACC}
_JOINT_KEYS = {"coeffs", "first_step", "last_step", "targets", "lower_tols", "upper_tols", "use_time"}
_CART_KEYS = {"timestep", "pos_coeffs", "rot_coeffs", "source_frame", "target_frame", "source_frame_offset_xyz",
              "source_frame_offset_wxyz", "target_frame_offset_xyz", "target_frame_offset_wxyz"}
_VEL_KEYS = {"first_step", "last_step", "max_displacement", "link"}
_COLL_KEYS = {"evaluator_type", "first_step", "last_step", "fixed_steps", "contact_test_type", "longest_valid_segment_length",
              "coeffs", "dist_pen", "pairs"}
_OPT_KEYS = ["improve_ratio_threshold", "min_trust_box_size", "min_approx_improve", "min_approx_improve_frac", "max_iter",
             "trust_shrink_ratio", "trust_expand_ratio", "cnt_tolerance", "max_merit_coeff_increases",
             "merit_coeff_increase_ratio", "max_time", "initial_merit_error_coeff", "inflate_constraints_individually",
             "trust_box_size"]


def _only(params, allowed):  # ensure_only_members, problem_description.cpp:32-51
    for k in params:
        if k not in allowed:
            raise ValueError(f'illegal field "{k}"')


def _req(v, key):
    if key not in v:
        raise ValueError(f"missing field: {key}")
    return v[key]


def _bcast(vals, n):  # checkParameterSize(..., apply_first=true)
    vals = list(np.atleast_1d(np.asarray(vals, float)))
    if len(vals) == 1 and n > 1:
        vals = vals * n
    if len(vals) != n:
        raise ValueError("parameter has the wrong size")
    return vals


def _term(v, role, T, D, link_of, root_frame, targets):
    typ = _req(v, "type")
    if v.get("use_time", False):
        raise ValueError(f"{typ}: use_time terms are not on the device path")
    params = v.get("params", {})
    if typ in _JOINT_KINDS:
        _only(params, _JOINT_KEYS)
        return problems.joint_term(_JOINT_KINDS[typ], role, D, params.get("first_step", 0), params.get("last_step", T - 1),
                                   coeffs=_bcast(params.get("coeffs", [1.0] * D), D), targets=_bcast(_req(params, "targets"), D),
                                   upper=_bcast(params.get("upper_tols", [0.0] * D), D),
                                   lower=_bcast(params.get("lower_tols", [0.0] * D), D), T=T)
    if typ == "cart_pose":
        _only(params, _CART_KEYS)
        if _req(params, "target_frame") != root_frame:
            raise ValueError(f'cart_pose: target_frame must be the static frame "{root_frame}" on the device path')
        slot = len(targets)
        targets.append(list(params.get("target_frame_offset_xyz", [0, 0, 0])) + list(params.get("target_frame_offset_wxyz", [1, 0, 0, 0])))
        return problems.cart_pose_term(role, params.get("timestep", T - 1), link_of(_req(params, "source_frame")), target_slot=slot,
                                       pos_coeffs=params.get("pos_coeffs", [1, 1, 1]), rot_coeffs=params.get("rot_coeffs", [1, 1, 1]),
                                       source_offset=list(params.get("source_frame_offset_xyz", [0, 0, 0])) +
                                       list(params.get("source_frame_offset_wxyz", [1, 0, 0, 0])))
    if typ == "cart_vel":
        _only(params, _VEL_KEYS)
        first, last = _req(params, "first_step"), _req(params, "last_step")
        if not (0 <= first < last <= T - 1):
            raise ValueError("cart_vel: invalid first_step / last_step")
        return problems.cart_vel_term(role, first, min(last, T - 2), link_of(_req(params, "link")), _req(params, "max_displacement"))
    if typ == "collision":
        _only(params, _COLL_KEYS)
        if "pairs" in params:
            raise ValueError("collision: per-pair overrides are not on the device path")
        first, last = params.get("first_step", 0), params.get("last_step", T - 1)
        if not (0 <= first <= last < T):
            raise ValueError("collision: invalid first_step / last_step")
        # the JSON path's default margin buffer is 0.5 m and cannot be overridden (problem_description.cpp:1625-1630, 1700-1711)
        return problems.collision_term(role, first, last, margin=_req(params, "dist_pen"), coeff=_req(params, "coeffs"), buffer=0.5,
                                       fixed_steps=params.get("fixed_steps", []), evaluator=params.get("evaluator_type", capi.COLL_DISCRETE),
                                       lvs=params.get("longest_valid_segment_length", 0.5))
    if typ in ("joint_jerk", "total_time", "dynamic_cart_pose"):
        raise ValueError(f'term type "{typ}" is not on the device path')
    raise ValueError(f"failed to construct cost named {typ}")  # problem_description.cpp:205-206


def from_json(doc, robot, start_states, link_names=None, root_frame="base_footprint", obstacles=None):
    """doc: JSON text or parsed dict.  robot: robots.* dict.  start_states: [B][D] (the environment's current joint values
    of every problem).  link_names: names of the robot's segments (default: the robot's own "link_names", else "link<i>")."""
    v = json.loads(doc) if isinstance(doc, str) else doc
    start = np.atleast_2d(np.asarray(start_states, float))
    B, D = start.shape
    names = link_names or robot.get("link_names") or [f"link{i}" for i in range(len(robot["segments"]))]

    def link_of(name):
        if name in names:
            return names.index(name)
        if name.startswith("link") and name[4:].isdigit() and int(name[4:]) < len(robot["segments"]):
            return int(name[4:])  # "link<i>": the i-th segment, whatever the robot calls it
        raise ValueError(f'link "{name}" is not part of the manipulator model')

    basic = _req(v, "basic_info")
    T = _req(basic, "n_steps")
    _req(basic, "manip")
    solver = basic.get("convex_solver", "AUTO_SOLVER")
    if solver not in ("OSQP", "AUTO_SOLVER"):
        if solver in ("GUROBI", "QPOASES", "BPMPD"):
            raise ValueError("the device path implements the OSQP-equivalent solver only")
        raise ValueError(f'invalid solver name:"{solver}"')
    if basic.get("use_time", False):
        raise ValueError("use_time problems are not on the device path")
    targets = []
    terms = [_term(c, capi.ROLE_COST, T, D, link_of, root_frame, targets) for c in v.get("costs", [])]
    terms += [_term(c, capi.ROLE_CNT, T, D, link_of, root_frame, targets) for c in v.get("constraints", [])]
    ii = _req(v, "init_info")
    kind = _req(ii, "type").lower()
    if kind == "stationary":
        init = np.repeat(start[:, None, :], T, axis=1)
    elif kind == "given_traj":
        data = np.asarray(_req(ii, "data"), float)
        if data.shape[0] != T:
            raise ValueError("given initialization traj has wrong length")
        init = np.repeat(data[None], B, axis=0)
    elif kind == "joint_interpolated":
        end = np.asarray(_req(ii, "endpoint"), float)
        if end.shape != (D,):
            raise ValueError(f"wrong number of dof values in initialization. expected {D} got {end.size}")
        init = problems.interpolate(start, np.repeat(end[None], B, axis=0), T)
    else:
        raise ValueError("init_info did not have a valid type from Json. Valid types are stationary, joint_interpolated, or given_traj")
    sqp = capi.default_sqp_params()
    for k in _OPT_KEYS:
        if k in v.get("opt_info", {}):
            setattr(sqp, k, type(getattr(sqp, k))(v["opt_info"][k]))
    cart = np.repeat(np.asarray(targets, float)[None], B, axis=0) if targets else None
    return capi.ProblemDesc(robot, T, terms, init, fixed_timesteps=basic.get("fixed_timesteps", []),
                            fixed_dofs=basic.get("fixed_dofs", []), cart_targets=cart, obstacles=obstacles, sqp=sqp)
