"""The convexify outputs against a plain high-precision numpy reference (tests/numpy_ref.py), at the branch points of
the kernel.

Every SQP iteration runs the convexify step: CartPose error and forward-difference Jacobian, CartVel rows, discrete and
continuous collision rows, the joint-term values and the exact cost_vals / cnt_viols of the merit decisions.  Elsewhere
the suite checks it against the CPU oracle, which restates the reference the way the kernel does, often line for line;
a mistake both make is invisible there.  Here the reference is numpy_ref: extended precision, no code shared with
either.  The cases are chosen to sit ON the branch points (exact activity ties, clamped sweep parameters, the fixed-step
filters, sub-segment counts at exact multiples, mask-word and chunk boundaries, rotation errors at 0, 2 pi / 3 and pi,
coincident centres, the LVS overflow), and every case asserts that it reached its edges: a case that silently stops
landing on its tie fails.  The census of edges is printed and asserted over the whole file.

The part without a marker runs without a GPU: numpy_ref against the oracle.  The GPU part holds the device against
numpy_ref and against the oracle on the same cases, and runs the overflow paths (convexify and solve).

Rotation errors of angle pi: a0 g0 and a0 (g0 - 2 pi sign g0) are the same rotation, and which one an fp64
implementation computes depends on the sign its rounding gives w.  The two are different linearisations, not one model
up to sign: the forward-difference Jacobian takes the 2 pi branch of its base, so its component along the axis is the
same in both and the component from the turning of the axis changes sign.  So within numpy_ref.PI_BAND of pi a CartPose
object must match one of the two numpy representatives, error and Jacobian together; everywhere else the one.
"""
import ctypes as C
import math
import time

import numpy as np
import pytest

import numpy_ref
from trajopt_b200 import api, capi, problems, robots
from trajopt_b200.capi import (COLL_CONTINUOUS, COLL_LVS_CONTINUOUS, COLL_LVS_DISCRETE, JOINT_FIXED,
                               JOINT_REVOLUTE, ROLE_CNT, ROLE_COST, TERM_JOINT_ACC, TERM_JOINT_POS, TERM_JOINT_VEL)
from test_shape_sweep import pr2_arm_6dof, rpr_arm

# the tolerances of test_gpu_parity.py
ROW_RTOL, JAC_RTOL, JAC_ATOL = 1e-10, 1e-6, 2e-9
COST_RTOL, COST_ATOL, VIOL_RTOL, VIOL_ATOL = 1e-12, 1e-14, 1e-9, 1e-12


# ---------------------------------------------------------------------------------------------------- robots
def spherebot7():
    """spherebot with seven spheres at dyadic offsets: every centre is exactly (q0 + cx, q1 + cy, cz)."""
    r = robots.spherebot()
    offs = [(0, 0, 0), (0.5, 0, 0), (-0.5, 0, 0), (0, 0.5, 0), (0, -0.5, 0), (0.25, 0.25, 0), (0, 0, 0.5)]
    r["spheres"] = [robots._sphere(2, c, rad) for c, rad in zip(offs, (0.5, 0.25, 0.25, 0.25, 0.25, 0.125, 0.25))]
    return r


def rr2():
    """Two revolute joints (z, then y) and a tool 0.4 m out: q = (theta, 0) turns the tool by exactly theta about z."""
    segs = [robots._seg(-1, JOINT_REVOLUTE, 0, (0, 0, 0.1), (0, 0, 1)),
            robots._seg(0, JOINT_REVOLUTE, 1, (0.5, 0, 0), (0, 1, 0)),
            robots._seg(1, JOINT_FIXED, -1, (0.4, 0, 0))]
    return dict(n_dof=2, segments=segs, lower=[-7.0, -7.0], upper=[7.0, 7.0], spheres=[robots._sphere(2, (0, 0, 0), 0.1)],
                link_names=["l0", "l1", "tool"], tool=2)


def _robot(D):
    return {2: spherebot7, 3: rpr_arm, 6: pr2_arm_6dof, 7: lambda: robots.pr2_arm("r"), 14: robots.pr2_dual_arm}[D]()


def _quat(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.r_[math.cos(ang / 2), math.sin(ang / 2) * axis]


def _rot(axis, ang):
    return robots._quat_to_rot(_quat(axis, ang))


def _vel(D, T):
    return problems.joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1)


# ---------------------------------------------------------------------------------------------------- the cases
# A case: (desc, x, edges) with edges a list of (census name, predicate on numpy_ref's info).
def _disc_tie():
    """spherebot at integer positions against obstacles of radius 4 at 3-4-5 distances: dist = 0.5 exactly.  Steps 1-2:
    margin + buffer = 0.25 + 0.25 = 0.5 (a tie: active); steps 3-4: 0.25 + (0.25 - 2^-54) = the double below 0.5 (dist
    one ulp above it: inactive)."""
    r = robots.spherebot()
    obs = np.array([[[3, 4, 0, 4.0], [-3, 4, 0, 4.0], [4, -3, 0, 4.0], [40, 0, 0, 1.0]]], float)
    x = np.zeros((2, 5, 2))
    x[1] += 1.0  # (the second trajectory is shifted with its world: the same ties)
    obs = np.concatenate([obs, obs + np.array([1, 1, 0, 0])])
    below = 0.25 - 2.0 ** -54
    terms = [_vel(2, 5), problems.collision_term(ROLE_CNT, 1, 2, margin=0.25, coeff=3.0, buffer=0.25),
             problems.collision_term(ROLE_COST, 3, 4, margin=0.25, coeff=2.0, buffer=below)]
    d = capi.ProblemDesc(r, 5, terms, x, fixed_timesteps=[0], obstacles=obs)
    return d, x, [("disc_tie_active", lambda i: i["disc_tie_active"] == 12),
                  ("disc_tie_one_ulp_above", lambda i: i["disc_tie_above"] == 12)]


def _disc_shape(O, L, D=2, shared=False, seed=0):
    """O obstacles against L spheres (D = 2: spherebot / spherebot7 on a grid), about half of them inside the reach."""
    rng = np.random.default_rng(seed)
    T, B = 3, 2
    if D == 2:
        r = spherebot7() if L == 7 else robots.spherebot()
        x = np.round(rng.uniform(-2, 2, (B, T, 2)) * 4) / 4
        lo, hi = np.array([-3, -3, -0.5]), np.array([3, 3, 0.5])
    else:
        r = _robot(D)
        lo_q, hi_q = np.array(r["lower"]), np.array(r["upper"])
        w = hi_q - lo_q
        x = rng.uniform(lo_q + 0.2 * w, hi_q - 0.2 * w, (B, T, D))
        cen = np.concatenate([robots.sphere_centers(r, q) for q in x.reshape(-1, D)])
        lo, hi = cen.min(0) - 0.3, cen.max(0) + 0.3
    n_w = 1 if shared else B
    obs = np.zeros((n_w, O, 4))
    obs[..., :3] = rng.uniform(lo, hi, (n_w, O, 3))
    obs[..., 3] = 0.125 if D == 2 else 0.05
    for w in range(n_w):  # (obstacle 0 touches sphere 0 at step 1: at least one active candidate in every world)
        c0, r0 = robots.sphere_centers(r, x[w, 1])[0], r["spheres"][0].radius
        obs[w, 0, :3] = c0 + np.array([0.6, 0.8, 0.0]) * (r0 + obs[w, 0, 3] + 0.02)
    L = len(r["spheres"])
    terms = [_vel(D, T), problems.collision_term(ROLE_CNT, 0, T - 1, margin=0.05, coeff=7.0, buffer=0.4 if D == 2 else 0.1,
                                               fixed_steps=[0])]
    d = capi.ProblemDesc(r, T, terms, x, fixed_timesteps=[0], obstacles=obs, obstacles_per_traj=not shared)
    name = f"disc_D{D}" if D != 2 else f"disc_O{O}_L{L}"
    return d, x, [(name, lambda i: 0 < i["disc_active"] < (T - 1) * B * O * L)] + \
        ([("disc_shared_world", lambda i: True)] if shared else [])


def _pair_desc(r, x, obs, terms, fixed=()):
    return capi.ProblemDesc(r, x.shape[1], [_vel(r["n_dof"], x.shape[1])] + terms, x, fixed_timesteps=list(fixed), obstacles=obs)


def _cast_steps():
    """spherebot steps of exactly lvs, 3 lvs and 4 lvs, and a stationary step (LVS_CONTINUOUS, lvs = 0.5)."""
    r = robots.spherebot()
    x = np.array([[[0, 0], [0.5, 0], [2.0, 0], [2.0, 0], [2.0, 2.0]]], float)
    obs = np.array([[[1.0, 0.9, 0, 0.3], [2.0, -1.0, 0, 0.3], [2.3, 1.0, 0, 0.3]]])
    t = problems.collision_term(ROLE_CNT, 0, 4, margin=0.1, coeff=5.0, buffer=0.4, evaluator=COLL_LVS_CONTINUOUS, lvs=0.5)
    return _pair_desc(r, x, obs, [t]), x, [
        ("cast_step_exactly_lvs", lambda i: i["cast_exact_lvs"] == 1 and i["cast_nsub"][0] == 1),
        ("cast_step_exactly_k_lvs", lambda i: i["cast_exact_multiple"] == 2 and i["cast_nsub"][1:] == [3, 1, 4]),
        ("cast_stationary", lambda i: i["cast_stationary"] == 1)]


def _cast_clamps(start_fixed, end_fixed):
    """Obstacles where the sweep parameter is exactly 0 (perpendicular at the start: wd = 0; behind the start: clamped)
    and exactly 1 (at the end), on the first and last sub-segments of 3 and on an interior one; with the start or the
    end of the pair fixed the Time0 / Time1 filters take them out, without they stay."""
    r = robots.spherebot()
    x = np.array([[[0, 0], [1.5, 0], [1.5, 0]]], float)
    obs = np.array([[[0, 0.9, 0, 0.3], [-0.9, 0, 0, 0.3], [1.5, 0.9, 0, 0.3], [2.4, 0, 0, 0.3], [0.5, 0.9, 0, 0.3]]])
    fixed = [0] if start_fixed else ([1] if end_fixed else [])
    t = problems.collision_term(ROLE_CNT, 0, 1, margin=0.1, coeff=5.0, buffer=0.2, evaluator=COLL_LVS_CONTINUOUS, lvs=0.5,
                                fixed_steps=fixed)
    d = capi.ProblemDesc(r, 3, [_vel(2, 3), t], x, fixed_timesteps=[0] if start_fixed else [], obstacles=obs)
    edges = [("cast_sc_0_interior", lambda i: i["sc_interior_clamp0"] > 0)]
    if start_fixed:
        edges.append(("time0_filter_fires", lambda i: i["time0_filtered"] == 2 and i["time1_kept"] == 2))
    elif end_fixed:
        edges.append(("time1_filter_fires", lambda i: i["time1_filtered"] == 2 and i["time0_kept"] == 2))
    else:
        edges.append(("time_filters_idle", lambda i: i["time0_kept"] == 2 and i["time1_kept"] == 2))
    return d, x, edges


def _cast_count(n_active):
    """One spherebot step pair with exactly n_active active contacts (every obstacle of a cluster inside the reach at
    every sub-segment): 63, 64 (one mask word), 65 (five sub-segments of 13), 128 (two of 64: the whole row block)."""
    O, step = {63: (63, 0.5), 64: (64, 0.5), 65: (13, 2.5), 128: (64, 1.0)}[n_active]
    r = robots.spherebot()
    x = np.array([[[0, 0], [step, 0]]], float)
    rng = np.random.default_rng(n_active)
    obs = np.zeros((1, O, 4))
    obs[0, :, :2] = rng.uniform([0, 0.9], [step, 1.1], (O, 2))
    obs[0, :, 3] = 0.2
    t = problems.collision_term(ROLE_COST, 0, 1, margin=0.1, coeff=2.0, buffer=3.0, evaluator=COLL_LVS_CONTINUOUS, lvs=0.5)
    return _pair_desc(r, x, obs, [t]), x, [(f"cast_{n_active}_active", lambda i: i["cast_active"] == [n_active])]


def _cast_mixed(D):
    """CONTINUOUS on the first step pairs and LVS_DISCRETE on the rest, fixed steps inside the ranges (D = 2 spherebot7,
    D = 7 PR2 arm: the two pair instances)."""
    rng = np.random.default_rng(D)
    T = 6
    if D == 2:
        r = spherebot7()
        x = np.cumsum(rng.uniform(-0.6, 0.6, (2, T, 2)), axis=1)
        obs = np.zeros((2, 6, 4))
        obs[..., :3] = rng.uniform([-1.5, -1.5, -0.3], [1.5, 1.5, 0.3], (2, 6, 3))
        obs[..., 3], lvs, buf = 0.2, 0.3, 0.3
    else:
        r = robots.pr2_arm("r")
        q0 = rng.uniform(np.array(r["lower"]) * 0.5, np.array(r["upper"]) * 0.5, (2, 7))
        x = q0[:, None] + np.cumsum(rng.uniform(-0.15, 0.15, (2, T, 7)), axis=1)
        cen = np.concatenate([robots.sphere_centers(r, q) for q in x.reshape(-1, 7)])
        obs = np.zeros((2, 8, 4))
        obs[..., :3] = rng.uniform(cen.min(0), cen.max(0), (2, 8, 3))
        obs[..., 3], lvs, buf = 0.05, 0.1, 0.1
    terms = [problems.collision_term(ROLE_CNT, 0, 3, margin=0.05, coeff=4.0, buffer=buf, evaluator=COLL_CONTINUOUS,
                                     fixed_steps=[0, 2]),
             problems.collision_term(ROLE_COST, 3, T - 1, margin=0.05, coeff=3.0, buffer=buf, evaluator=COLL_LVS_DISCRETE,
                                     lvs=lvs, fixed_steps=[4])]
    d = _pair_desc(r, x, obs, terms, fixed=[0])
    return d, x, [(f"cast_mixed_D{D}", lambda i: sum(i["cast_active"]) > 0 and max(i["cast_nsub"]) > 1)]


def _cast_rr2():
    """rr2 with spheres off their link origins (a revolute link turns them between the ends of a sub-segment, so the
    reference points of the two gradients differ), CONTINUOUS and LVS_CONTINUOUS with both ends free."""
    r = rr2()
    r["spheres"] = [robots._sphere(1, (0.2, 0.05, 0), 0.1), robots._sphere(2, (0.1, 0, 0.05), 0.08)]
    x = np.array([[[0.0, 0.0], [0.9, 0.4], [1.6, -0.3], [2.2, 0.2]], [[-1.0, 0.3], [-0.2, -0.5], [0.5, 0.1], [1.2, 0.6]]])
    rng = np.random.default_rng(11)
    cen = np.concatenate([robots.sphere_centers(r, q) for q in x.reshape(-1, 2)])
    obs = np.zeros((2, 10, 4))
    obs[..., :3] = rng.uniform(cen.min(0) - 0.1, cen.max(0) + 0.1, (2, 10, 3))
    obs[..., 3] = 0.1
    terms = [problems.collision_term(ROLE_CNT, 0, 2, margin=0.05, coeff=4.0, buffer=0.2, evaluator=COLL_CONTINUOUS),
             problems.collision_term(ROLE_COST, 2, 3, margin=0.05, coeff=3.0, buffer=0.2, evaluator=COLL_LVS_CONTINUOUS,
                                     lvs=0.3)]
    return _pair_desc(r, x, obs, terms), x, [("cast_revolute_offset_spheres", lambda i: sum(i["cast_active"]) >= 10)]


def _coincident():
    """A spherebot centre exactly on an obstacle centre (discrete), and a swept segment through one (continuous)."""
    r = robots.spherebot()
    x = np.array([[[1, 2], [1, 2], [3, 2]]], float)
    obs = np.array([[[1, 2, 0, 0.5], [2, 2, 0, 0.25], [5, 5, 0, 0.5]]])
    disc = capi.ProblemDesc(r, 3, [_vel(2, 3), problems.collision_term(ROLE_CNT, 0, 2, margin=0.1, coeff=2.0, buffer=0.1)],
                            x, obstacles=obs)
    cast = _pair_desc(r, x, obs, [problems.collision_term(ROLE_CNT, 0, 2, margin=0.1, coeff=2.0, buffer=0.1,
                                                          evaluator=COLL_CONTINUOUS)])
    return [(disc, x, [("coincident_discrete", lambda i: i["coincident_discrete"] == 2)]),
            (cast, x, [("coincident_cast", lambda i: i["coincident_cast"] > 0)])]


# the rotation errors of the CartPose cases (rad): identity, tiny, both sides of the trace = 0 switch of the quaternion
# extraction (angle 2 pi / 3), a perturbation that crosses pi, and pi itself
ANGLES = [0.0, 1e-9, 2 * math.pi / 3 - 1e-3, 2 * math.pi / 3 + 1e-3, math.pi - 1e-6, math.pi]


def _cart_rr2():
    """rr2 with one CartPose object per step (14 > the 8 warps): the first six at the angles of ANGLES about z (fixed
    target_pose), then targets given as -q and 2q, a rotated source_offset, coefficient subsets with negative
    coefficients, and per-trajectory target slots next to the fixed targets; as costs and as constraints."""
    r = rr2()
    T, tool = 14, r["tool"]
    x = np.zeros((2, T, 2))
    x[:, :6, 0] = ANGLES
    x[1, :6, 0] *= -1
    rng = np.random.default_rng(3)
    x[:, 6:] = rng.uniform(-2.5, 2.5, (2, T - 6, 2))
    terms = [_vel(2, T + 2)]
    p_t = (0.9, 0.0, 0.1)
    for t in range(6):
        terms.append(problems.cart_pose_term(ROLE_CNT if t % 2 else ROLE_COST, t, tool, target_pose=(*p_t, 1, 0, 0, 0)))
    q = _quat((0.3, -0.2, 1.0), 0.7)
    terms.append(problems.cart_pose_term(ROLE_CNT, 6, tool, target_pose=(0.5, 0.2, 0.0, *(-q))))
    terms.append(problems.cart_pose_term(ROLE_COST, 7, tool, target_pose=(0.5, 0.2, 0.0, *(2 * q))))
    off = (0.05, -0.02, 0.03, *_quat((1, 1, 0), 0.4))
    terms.append(problems.cart_pose_term(ROLE_CNT, 8, tool, target_pose=(0.4, 0.1, 0.2, *q), source_offset=off))
    terms.append(problems.cart_pose_term(ROLE_COST, 9, tool, target_pose=(0.4, 0.1, 0.2, *q), pos_coeffs=(1, 0, -2),
                                         rot_coeffs=(0, -1.5, 3)))
    terms.append(problems.cart_pose_term(ROLE_CNT, 10, tool, target_pose=(0.4, 0.1, 0.2, *q), pos_coeffs=(0, -0.5, 0),
                                         rot_coeffs=(2, 0, 0), source_offset=off))
    for k, t in enumerate(range(11, T)):
        terms.append(problems.cart_pose_term(ROLE_CNT if k % 2 else ROLE_COST, t, tool, target_slot=k))
    tg = np.zeros((2, 5, 7))
    for b in range(2):
        for k in range(3):
            tg[b, k, :3] = rng.uniform(-0.5, 0.5, 3)
            tg[b, k, 3:] = _quat(rng.standard_normal(3), rng.uniform(0, 3))
    # two more steps whose error rotation is pi - 1e-6 and pi - 1e-4 about (1, -1, 0) / sqrt 2: the two largest diagonal
    # entries tie, so the perturbed states take the other branch of the quaternion extraction and their axis comes out
    # flipped (calcJacobianTransformErrorDiff's flip)
    x = np.concatenate([x, rng.uniform(-2.5, 2.5, (2, 2, 2))], axis=1)
    for k, (t, ang) in enumerate(((T, math.pi - 1e-6), (T + 1, math.pi - 1e-4))):
        terms.append(problems.cart_pose_term(ROLE_CNT, t, tool, target_slot=3 + k))
        for b in range(2):
            R, p = robots.fk_numpy(r, x[b, t])[tool]
            tg[b, 3 + k, :3], tg[b, 3 + k, 3:] = p, robots.rot_to_wxyz(R @ _rot((1, -1, 0), ang).T)
    d = capi.ProblemDesc(r, T + 2, terms, x, cart_targets=tg)
    return d, x, _angle_edges("rr2") + [("cart_axis_flip", lambda i: i["cart_axis_flips"] > 0)]


def _angle_edges(tag):
    def near(a):
        return lambda i: any(abs(abs(g) - a) < 1e-13 for g in i["cart_angle"])
    return [(f"{tag}_angle_0", near(0.0)),
            (f"{tag}_angle_1e-9", near(1e-9)),
            (f"{tag}_angle_2pi/3-1e-3", near(2 * math.pi / 3 - 1e-3)),
            (f"{tag}_angle_2pi/3+1e-3", near(2 * math.pi / 3 + 1e-3)),
            (f"{tag}_angle_pi-1e-6", near(math.pi - 1e-6)),
            (f"{tag}_angle_pi", lambda i: any(abs(abs(g) - math.pi) < 1e-15 for g in i["cart_angle"]))]


def _cart_pr2():
    """The PR2 arm with targets at the rotation errors of ANGLES about a generic axis (fp64 targets: at pi the sign of w
    is a rounding), a rotated source_offset on half of them, and CartVel on a link the wrist does not move."""
    r = robots.pr2_arm("r")
    T, D, tool = len(ANGLES), 7, r["tool"]
    rng = np.random.default_rng(5)
    x = rng.uniform(np.array(r["lower"]) * 0.6, np.array(r["upper"]) * 0.6, (2, T, D))
    off = (0.02, 0.0, -0.01, *_quat((0, 1, 1), 0.3))
    terms = [_vel(D, T)]
    tg = np.zeros((2, T, 7))
    for t, ang in enumerate(ANGLES):
        so = off if t % 2 else (0, 0, 0, 1, 0, 0, 0)
        terms.append(problems.cart_pose_term(ROLE_CNT if t % 2 else ROLE_COST, t, tool, target_slot=t, source_offset=so))
        for b in range(2):
            R, p = robots.fk_numpy(r, x[b, t])[tool]
            Ro = robots._quat_to_rot(so[3:])
            Rs, ps = R @ Ro, R @ np.array(so[:3]) + p
            Rt = Rs @ _rot(rng.standard_normal(3), ang).T  # target^-1 source = the rotation of angle `ang`
            tg[b, t, :3], tg[b, t, 3:] = ps + rng.uniform(-0.1, 0.1, 3), robots.rot_to_wxyz(Rt)
    elbow = r["link_names"].index("r_elbow_flex_link")
    terms.append(problems.cart_vel_term(ROLE_CNT, 0, T - 2, elbow, 0.05))
    d = capi.ProblemDesc(r, T, terms, x, fixed_timesteps=[0], cart_targets=tg)
    return d, x, _angle_edges("pr2") + [("cartvel_joint_mask", lambda i: True)]


def _cart_vel_spherebot():
    """CartVel of spherebot's x link (joint 1 does not move it) on every pair, the first next to the fixed step 0."""
    r = robots.spherebot()
    x = np.array([[[0, 0], [0.25, 1.0], [1.0, -0.5], [1.0, -0.5]]], float)
    terms = [_vel(2, 4), problems.cart_vel_term(ROLE_CNT, 0, 2, 0, 0.3), problems.cart_vel_term(ROLE_COST, 0, 2, 2, 0.5)]
    return capi.ProblemDesc(r, 4, terms, x, fixed_timesteps=[0]), x, [("cartvel_pair_next_to_fixed", lambda i: True)]


def _joint_terms():
    """Every joint-term flavour (Pos / Vel / Acc, Eq / Ineq, cost / constraint: the Eq constraint's c e^2 value)."""
    r = robots.pr2_arm("r", with_spheres=False)
    D, T = 7, 6
    rng = np.random.default_rng(9)
    x = rng.uniform(-1, 1, (2, T, D))
    terms = [problems.joint_term(TERM_JOINT_POS, ROLE_CNT, D, 1, 2, coeffs=3.0, targets=0.2),
             problems.joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1, coeffs=2.0, targets=0.01),
             problems.joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1, coeffs=1.0, upper=0.05, lower=-0.05),
             problems.joint_term(TERM_JOINT_VEL, ROLE_CNT, D, 0, T - 1, coeffs=0.5, upper=0.1, lower=-0.2),
             problems.joint_term(TERM_JOINT_ACC, ROLE_CNT, D, 1, T - 1, coeffs=1.5, targets=-0.1)]
    return capi.ProblemDesc(r, T, terms, x, fixed_timesteps=[0]), x, [("joint_terms", lambda i: True)]


def _config(name):
    d = {"cfg1": lambda: problems.config1(B=3, T=12), "cfg2": lambda: problems.config2(B=3, T=12),
         "cfg3": lambda: problems.config3(B=2, T=12, via_every=4),
         "cfg3_lvs_discrete": lambda: problems.config3(B=2, T=12, via_every=4, evaluator=COLL_LVS_DISCRETE),
         "cfg4": lambda: problems.config4(B=2, T=8), "variants": lambda: problems.config_variants(B=3, T=10)}[name]()
    x = d.init_traj + 0.05 * np.random.default_rng(7).standard_normal(d.init_traj.shape)
    return d, x, []


def _cases():
    c = {k: (lambda k=k: _config(k)) for k in ("cfg1", "cfg2", "cfg3", "cfg3_lvs_discrete", "cfg4", "variants")}
    c["disc_tie"] = _disc_tie
    for O in (1, 31, 32, 33, 63, 64):
        for L in (1, 7):
            c[f"disc_O{O}_L{L}"] = lambda O=O, L=L: _disc_shape(O, L, seed=O * 10 + L)
    for D, O in ((7, 33), (3, 20), (6, 9), (14, 8)):  # (odd D: staged 16-byte row stores; even D: scalar stores)
        c[f"disc_D{D}"] = lambda D=D, O=O: _disc_shape(O, 0, D=D, seed=D)
    c["disc_shared_world"] = lambda: _disc_shape(64, 7, shared=True, seed=1)
    c["cast_steps"] = _cast_steps
    c["cast_clamp_start_fixed"] = lambda: _cast_clamps(True, False)
    c["cast_clamp_end_fixed"] = lambda: _cast_clamps(False, True)
    c["cast_clamp_free"] = lambda: _cast_clamps(False, False)
    for n in (63, 64, 65, 128):
        c[f"cast_{n}_active"] = lambda n=n: _cast_count(n)
    c["cast_mixed_D2"] = lambda: _cast_mixed(2)
    c["cast_mixed_D7"] = lambda: _cast_mixed(7)
    c["cast_rr2"] = _cast_rr2
    c["coincident_discrete"] = lambda: _coincident()[0]
    c["coincident_cast"] = lambda: _coincident()[1]
    c["cart_rr2"] = _cart_rr2
    c["cart_pr2"] = _cart_pr2
    c["cart_vel_spherebot"] = _cart_vel_spherebot
    c["joint_terms"] = _joint_terms
    return c


CASES = _cases()
EDGES = ["disc_tie_active", "disc_tie_one_ulp_above", "disc_shared_world", "cast_step_exactly_lvs", "cast_step_exactly_k_lvs",
         "cast_stationary", "cast_sc_0_interior", "time0_filter_fires", "time1_filter_fires", "time_filters_idle",
         "cast_mixed_D2", "cast_mixed_D7", "cast_revolute_offset_spheres", "cart_axis_flip", "coincident_discrete", "coincident_cast", "cartvel_joint_mask",
         "cartvel_pair_next_to_fixed", "joint_terms"] + \
    [f"disc_O{O}_L{L}" for O in (1, 31, 32, 33, 63, 64) for L in (1, 7)] + [f"disc_D{D}" for D in (7, 3, 6, 14)] + \
    [f"cast_{n}_active" for n in (63, 64, 65, 128)] + [e for tag in ("rr2", "pr2") for e, _ in _angle_edges(tag)] + \
    ["lvs_overflow_contacts", "lvs_overflow_subsegments", "lvs_overflow_solve"]


class _Built(dict):
    def __missing__(self, name):
        d, x, edges = CASES[name]()
        ref, info = numpy_ref.convexify(d, x)
        self[name] = (d, x, edges, ref, info)
        return self[name]


BUILT = _Built()
CENSUS = {"cpu": set(), "gpu": set()}


def _reach(name, side):
    """The case's edges, each asserted on numpy_ref's account of the input, into the census of `side`."""
    d, x, edges, ref, info = BUILT[name]
    for e, pred in edges:
        assert pred(info), (name, e, {k: v for k, v in info.items() if k != "cart_alt"})
        CENSUS[side].add(e)


# ---------------------------------------------------------------------------------------------------- comparisons
def _cart_objects(d):
    """(first row, number of rows) of every CartPose object, in row order."""
    out, r = [], 0
    for t in d.terms:
        if t.kind == capi.TERM_CART_POSE:
            out.append((r, len(numpy_ref.cart_idx(t))))
            r += len(numpy_ref.cart_idx(t))
        elif t.kind == capi.TERM_CART_VEL:
            r += 6 * (t.last_step - t.first_step + 1)
    return out


def assert_matches_numpy(d, got, ref, info, bs=None, exact_geometry=False):
    """got (device or oracle) against numpy_ref at the tolerances of test_gpu_parity.py; rotation errors within
    PI_BAND of pi may take the other representative (module docstring), error and Jacobian of the object together."""
    bs = list(range(d.B)) if bs is None else list(bs)
    ce, cj = got["cart_err"][bs].copy(), got["cart_jac"][bs].copy()
    re_, rj = ref["cart_err"][bs].copy(), ref["cart_jac"][bs].copy()
    for k, b in enumerate(bs):
        for r0, n in _cart_objects(d):
            alt = info["cart_alt"].get((b, r0))
            if alt is None:
                continue
            ea, ja = alt
            ok = np.allclose(ce[k, r0:r0 + n], ea, rtol=ROW_RTOL, atol=1e-9) and \
                np.allclose(cj[k, r0:r0 + n, :ja.shape[1]], ja, rtol=JAC_RTOL, atol=JAC_ATOL)
            if ok:  # the other representative: held against that one at the usual tolerances
                re_[k, r0:r0 + n], rj[k, r0:r0 + n, :ja.shape[1]] = ea, ja
    np.testing.assert_allclose(ce, re_, rtol=ROW_RTOL, atol=1e-12)
    np.testing.assert_allclose(cj, rj, rtol=JAC_RTOL, atol=JAC_ATOL)
    np.testing.assert_allclose(got["cost_vals"][bs], ref["cost_vals"][bs], rtol=COST_RTOL, atol=COST_ATOL)
    np.testing.assert_allclose(got["cnt_viols"][bs], ref["cnt_viols"][bs], rtol=VIOL_RTOL, atol=VIOL_ATOL)
    gr, rr = got["coll_rows"][bs], ref["coll_rows"][bs]
    assert gr.shape == rr.shape
    assert np.isfinite(gr).all()
    assert ((gr[..., -1] != 0) == (rr[..., -1] != 0)).all(), np.argwhere((gr[..., -1] != 0) != (rr[..., -1] != 0))[:8]
    # spherebot on integer and dyadic geometry: distances and normals are exact or within an ulp in fp64
    np.testing.assert_allclose(gr, rr, rtol=0 if exact_geometry else ROW_RTOL, atol=4e-16 if exact_geometry else 1e-12)


def _exact(name):
    return name.startswith(("disc_tie", "cast_steps", "cast_clamp", "coincident"))


# ====================================================================================================== CPU part
@pytest.mark.parametrize("name", list(CASES))
def test_numpy_reference_matches_oracle(oracle, name):
    d, x, edges, ref, info = BUILT[name]
    got = oracle.convexify_batch(d, x)
    assert_matches_numpy(d, got, ref, info, exact_geometry=_exact(name))
    _reach(name, "cpu")


def test_cart_jacobian_against_central_differences():
    """The forward-difference rotation rows of numpy_ref against scipy's rotation vector, central differences, away
    from pi (an independent check of the quotient and of its flip / wrap rule where both must agree)."""
    for name in ("cart_rr2", "cart_pr2"):
        d, x, _, _, _ = BUILT[name]
        n = 0
        for b in range(d.B):
            for tm in d.terms:
                if tm.kind != capi.TERM_CART_POSE:
                    continue
                tgt = d.cart_targets[b, tm.target_slot] if tm.target_slot >= 0 else list(tm.target_pose)
                q = x[b, tm.first_step]
                err, J, g0, _ = numpy_ref.cart_pose_rows(d.robot_spec, tm, tgt, q)
                if abs(float(g0)) > math.pi - 1e-3:
                    continue
                rv, Jc = numpy_ref.rotvec_error_central(d.robot_spec, tm, tgt, q)
                np.testing.assert_allclose(np.array(err[3:], float), rv, rtol=0, atol=1e-12)
                np.testing.assert_allclose(np.array(J[3:], float), Jc, rtol=0, atol=1e-4)
                n += 1
        assert n >= 8


# -------------------------------------------------------------------------------------------- LVS overflow inputs
def _overflow_contacts():
    """B = 3 spherebot, 64 obstacles clustered by the path, initial trajectories stationary (row block: 128 rows per
    pair); at x, trajectory 0 steps 1.5 = 3 lvs: 192 active contacts in one pair.  Trajectories 1 and 2 stay inside."""
    r = robots.spherebot()
    init = np.zeros((3, 3, 2))
    init[:, :, 1] = np.array([0.0, 5.0, -5.0])[:, None]
    x = init.copy()
    x[0, 2, 0] = 1.5
    x[1, 2, 0], x[2, 1, 1] = 0.4, -5.2
    rng = np.random.default_rng(1)
    obs = np.zeros((3, 64, 4))
    obs[..., :2] = init[:, :1, :] + rng.uniform([0, 0.9], [1.5, 1.1], (3, 64, 2))
    obs[..., 3] = 0.2
    t = problems.collision_term(ROLE_CNT, 0, 2, margin=0.1, coeff=2.0, buffer=3.0, evaluator=COLL_LVS_CONTINUOUS, lvs=0.5)
    return _pair_desc(r, init, obs, [t]), x


LVS_TINY = 2.0 ** -15


def _overflow_subsegments():
    """Trajectory 0 steps 1.0 at lvs = 2^-15: 32768 sub-segments, one more than the 15-bit key holds."""
    r = robots.spherebot()
    init = np.zeros((3, 2, 2))
    init[:, :, 1] = np.array([0.0, 3.0, -3.0])[:, None]
    x = init.copy()
    x[0, 1, 0] = 1.0
    x[1, 1, 0] = 1e-5
    obs = np.zeros((3, 2, 4))
    obs[:, 0, 1] = init[:, 0, 1] + 0.8  # (a contact of trajectories 1 and 2; trajectory 0 has none, only its length)
    obs[0, 0, :2] = [30, -30]
    obs[:, 1, :2] = [30, 30]
    obs[..., 3] = 0.25
    t = problems.collision_term(ROLE_CNT, 0, 1, margin=0.1, coeff=2.0, buffer=0.1, evaluator=COLL_LVS_CONTINUOUS,
                                lvs=LVS_TINY)
    return _pair_desc(r, init, obs, [t]), x


def _overflow_solve():
    """B = 3 where only trajectory 0 outgrows its row block at the initial evaluation: 70 sub-segments x 64 obstacles,
    every one inside the reach (4480 contacts; the row block stops at 4096).  Trajectories 1 and 2 move little, one
    obstacle of their worlds near them."""
    r = robots.spherebot()
    T = 4
    init = np.zeros((3, T, 2))
    init[0, :, 0] = [0.0, 0.7, 0.7, 0.7]
    init[1, :, :] = np.c_[np.linspace(5, 5.02, T), np.zeros(T)]
    init[2, :, :] = np.c_[np.zeros(T), np.linspace(-5, -5.02, T)]
    rng = np.random.default_rng(2)
    obs = np.zeros((3, 64, 4))
    obs[0, :, :2] = rng.uniform([0.2, 0.85], [0.5, 0.95], (64, 2))
    obs[1:, :, :2] = rng.uniform([20, 20], [30, 30], (2, 64, 2))
    obs[1, 0, :2], obs[2, 0, :2] = [5.0, 0.85], [0.8, -5.0]
    obs[..., 3] = 0.3
    t = problems.collision_term(ROLE_CNT, 0, T - 1, margin=0.05, coeff=10.0, buffer=0.3, evaluator=COLL_LVS_CONTINUOUS,
                                lvs=0.01, fixed_steps=[0])
    return capi.ProblemDesc(r, T, [_vel(2, T), t], init, fixed_timesteps=[0], obstacles=obs)


def test_overflow_inputs_reach_their_edges(oracle):
    """The overflow inputs do what they are built for (numpy_ref's account): trajectory 0 alone overflows, by contacts
    (192 > 128), by sub-segments (32768 > 32767), and at the initial trajectory of the solve (4480 > 4096); the other
    trajectories' rows are the oracle's."""
    d, x = _overflow_contacts()
    assert numpy_ref.cast_rows_per_pair(d) == 128
    ref, info = numpy_ref.convexify(d, x)
    assert info["overflow"] == [0] and 192 in info["cast_active"], info["cast_active"]
    assert_matches_numpy(d, oracle.convexify_batch(d, x, 1, 3), ref, info, bs=[1, 2], exact_geometry=True)
    d, x = _overflow_subsegments()
    ref, info = numpy_ref.convexify(d, x)
    assert info["overflow"] == [0] and max(info["cast_nsub"]) == 32768
    assert_matches_numpy(d, oracle.convexify_batch(d, x, 1, 3), ref, info, bs=[1, 2])
    d = _overflow_solve()
    assert numpy_ref.cast_rows_per_pair(d) == 4096
    ref, info = numpy_ref.convexify(d, d.init_traj, bs=[0])
    assert info["overflow"] == [0] and max(info["cast_active"]) == 4480, info["cast_active"]
    ref = oracle.solve_batch(d.slice(1, 3))
    assert (ref["status"] != capi.OPT_INVALID).all()
    CENSUS["cpu"] |= {"lvs_overflow_contacts", "lvs_overflow_subsegments", "lvs_overflow_solve"}


def test_census_cpu():
    """Every edge of the catalogue was reached by the CPU part (cases the run did not cover are built here)."""
    _census("cpu", lambda name: _reach(name, "cpu"))


def _census(side, visit):
    for name in CASES:
        visit(name)
    if "lvs_overflow_solve" not in CENSUS[side] and side == "cpu":
        import oracle_lib
        test_overflow_inputs_reach_their_edges(oracle_lib)
    print(f"\nconvexify edge census ({side}):")
    for e in EDGES:
        print(f"  {'reached' if e in CENSUS[side] else 'MISSED ':<8} {e}")
    missed = [e for e in EDGES if e not in CENSUS[side]]
    assert not missed, missed


# ====================================================================================================== GPU part
def _convexify_raw(p, x):
    """tb200_convexify_batch with its return code and message (api.Problem.convexify raises on an error, and the rows
    of the other trajectories are what an overflow test needs)."""
    L, d = p.layout, p.desc
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = dict(cart_err=np.zeros((d.B, max(L.n_cart_rows, 1))),
               cart_jac=np.zeros((d.B, max(L.n_cart_rows, 1), max(L.cart_jac_stride, 1))),
               coll_rows=np.zeros((d.B, max(L.n_coll_cand, 1), L.coll_row_stride)),
               cost_vals=np.zeros((d.B, max(L.n_costs, 1))), cnt_viols=np.zeros((d.B, max(L.n_cnts, 1))))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    co = capi.ConvexifyOut(*[dp(out[k]) for k in ("cart_err", "cart_jac", "coll_rows", "cost_vals", "cnt_viols")])
    rc = p.lib.tb200_convexify_batch(p.handle, dp(x), C.byref(co))
    msg = p.lib.tb200_last_error().decode() if rc else ""
    for k, n in (("cart_err", L.n_cart_rows), ("cart_jac", L.n_cart_rows), ("coll_rows", L.n_coll_cand),
                 ("cost_vals", L.n_costs), ("cnt_viols", L.n_cnts)):
        out[k] = out[k][:, :n]
    return rc, msg, out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_matches_numpy_and_oracle(oracle, name):
    d, x, edges, ref, info = BUILT[name]
    p = api.Problem(d)
    try:
        rc, msg, got = _convexify_raw(p, x)
    finally:
        p.close()
    assert rc == 0, msg
    assert_matches_numpy(d, got, ref, info, exact_geometry=_exact(name))
    want = oracle.convexify_batch(d, x)
    np.testing.assert_allclose(got["cart_jac"], want["cart_jac"], rtol=JAC_RTOL, atol=JAC_ATOL)
    np.testing.assert_allclose(got["cost_vals"], want["cost_vals"], rtol=COST_RTOL, atol=COST_ATOL)
    np.testing.assert_allclose(got["cnt_viols"], want["cnt_viols"], rtol=VIOL_RTOL, atol=VIOL_ATOL)
    if got["coll_rows"].size:
        np.testing.assert_allclose(got["coll_rows"], want["coll_rows"], rtol=ROW_RTOL, atol=1e-12)
    if not info["cart_alt"]:  # (at pi the device and the oracle may each take either representative)
        np.testing.assert_allclose(got["cart_err"], want["cart_err"], rtol=ROW_RTOL, atol=1e-12)
    _reach(name, "gpu")


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["contacts", "subsegments"])
def test_device_convexify_overflow(oracle, which):
    """A step pair beyond the row block (192 active contacts in 128 rows) or beyond 32767 sub-segments: the call
    returns TB200_ERR_UNSUPPORTED with its message, and the rows of the other trajectories are numpy_ref's."""
    d, x = _overflow_contacts() if which == "contacts" else _overflow_subsegments()
    ref, info = numpy_ref.convexify(d, x, bs=[1, 2])
    p = api.Problem(d)
    try:
        t0 = time.perf_counter()
        rc, msg, got = _convexify_raw(p, x)
        wall = time.perf_counter() - t0
        dev_ms = p.timing()["convexify_ms"]
    finally:
        p.close()
    print(f"\noverflow by {which}: convexify kernel {dev_ms:.2f} ms on the device, {wall * 1e3:.1f} ms for the call")
    assert rc == capi.ERR_UNSUPPORTED, (rc, msg)
    assert "1 trajectories have a step pair with more than 128 active continuous-collision contacts" in msg, msg
    assert "more than 32767 longest-valid-segment sub-segments" in msg and "OPT_FAILED" in msg, msg
    assert_matches_numpy(d, got, ref, info, bs=[1, 2], exact_geometry=which == "contacts")
    assert dev_ms < 3000.0
    CENSUS["gpu"].add(f"lvs_overflow_{which}")


@pytest.mark.gpu
def test_device_solve_overflow_ends_only_its_trajectory(oracle):
    """B = 3, only trajectory 0 outgrows its row block at the initial evaluation: the solve returns
    TB200_ERR_UNSUPPORTED, trajectory 0 ends OPT_FAILED, and trajectories 1 and 2 are the oracle's solve of that
    slice of the batch."""
    d = _overflow_solve()
    p = api.Problem(d)
    try:
        buf, res = capi.alloc_results(d.B, d.T, d.D, p.layout.n_costs, p.layout.n_cnts)
        rc = p.lib.tb200_solve_batch(p.handle, C.byref(res))
        msg = p.lib.tb200_last_error().decode() if rc else ""
    finally:
        p.close()
    assert rc == capi.ERR_UNSUPPORTED and "1 trajectories have a step pair with more than 4096" in msg, (rc, msg)
    assert buf["status"][0] == capi.OPT_FAILED, buf["status"]
    ref = oracle.solve_batch(d.slice(1, 3))
    assert (buf["status"][1:] == ref["status"]).all(), (buf["status"], ref["status"])
    assert (buf["n_qp_solves"][1:] == ref["n_qp_solves"]).all(), (buf["n_qp_solves"], ref["n_qp_solves"])
    np.testing.assert_allclose(buf["total_cost"][1:], ref["total_cost"], atol=1e-6)
    np.testing.assert_allclose(buf["x"][1:], ref["x"], atol=1e-5)
    CENSUS["gpu"].add("lvs_overflow_solve")


@pytest.mark.gpu
def test_census_gpu(oracle):
    """Every edge of the catalogue was reached on the device (cases the run did not cover are run here)."""
    def visit(name):
        if any(e not in CENSUS["gpu"] for e, _ in BUILT[name][2]):
            test_device_matches_numpy_and_oracle(oracle, name)
    for which in ("contacts", "subsegments"):
        if f"lvs_overflow_{which}" not in CENSUS["gpu"]:
            test_device_convexify_overflow(oracle, which)
    if "lvs_overflow_solve" not in CENSUS["gpu"]:
        test_device_solve_overflow_ends_only_its_trajectory(oracle)
    _census("gpu", visit)
