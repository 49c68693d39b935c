"""Synthetic problem sets of BASELINE.json `configs` (definitions: SURVEY.md §8d).

configs[k] uses numpy.random.default_rng(20260923 + k).  The generated arrays are the byte-identical
inputs fed to both the CUDA path and the CPU oracle.
"""
import numpy as np

from . import capi, robots
from .capi import (COLL_DISCRETE, COLL_LVS_CONTINUOUS, ROLE_CNT, ROLE_COST, TERM_AVOID_SINGULARITY, TERM_CART_POSE,
                   TERM_CART_VEL, TERM_COLLISION, TERM_JOINT_ACC, TERM_JOINT_POS, TERM_JOINT_VEL, ProblemDesc, Term)

SEED = 20260923


def hatch_steps(kind, first, last, T):
    """Step clamping of Joint{Pos,Vel,Acc}TermInfo::hatch (problem_description.cpp:1078-1106, 1197-1224,
    1393-1421): last_step <= -1 means "to the end"; vel needs >= 2 steps, acc >= 3."""
    if last <= -1:
        last = T - 1
    order = kind - TERM_JOINT_POS
    if (T - 1 - order) <= first:
        first = T - 1 - order
    if (T - 1) <= last:
        last = T - 1
    if order > 0 and last == first:
        last += order
    if last < first:
        first, last = last, first
    return first, last


def joint_term(kind, role, D, first, last, coeffs=1.0, targets=0.0, upper=0.0, lower=0.0, T=None):
    if T is not None:
        first, last = hatch_steps(kind, first, last, T)
    t = Term()
    t.kind, t.role, t.first_step, t.last_step = kind, role, first, last
    for name, v in (("coeffs", coeffs), ("targets", targets), ("upper_tols", upper), ("lower_tols", lower)):
        arr = np.broadcast_to(np.asarray(v, float), (D,))
        getattr(t, name)[:D] = arr.tolist()
    return t


def cart_pose_term(role, timestep, link, target_slot=-1, target_pose=None, pos_coeffs=(1, 1, 1), rot_coeffs=(1, 1, 1),
                   source_offset=(0, 0, 0, 1, 0, 0, 0)):
    t = Term()
    t.kind, t.role, t.first_step, t.last_step = TERM_CART_POSE, role, timestep, timestep
    t.link, t.target_slot = link, target_slot
    t.source_offset[:] = source_offset
    t.target_pose[:] = target_pose if target_pose is not None else (0, 0, 0, 1, 0, 0, 0)
    t.pos_coeffs[:] = pos_coeffs
    t.rot_coeffs[:] = rot_coeffs
    return t


def avoid_singularity_term(role, first, last, link, coeff=1.0, lam=0.1):
    """AvoidSingularityTermInfo (problem_description.cpp:1900-1939): one object per step first..last on the smallest
    singular value of `link`'s geometric Jacobian; an ABS cost (role COST) or an INEQ constraint (role CNT)."""
    t = Term()
    t.kind, t.role, t.first_step, t.last_step = TERM_AVOID_SINGULARITY, role, first, last
    t.link, t.target_slot = link, -1
    t.coeffs[0] = coeff
    t.lambda_ = lam
    return t


def cart_vel_term(role, first, last, link, max_displacement):
    """CartVelTermInfo (problem_description.cpp:989-1057): one object per step pair first..last (pair t = (t, t+1))."""
    t = Term()
    t.kind, t.role, t.first_step, t.last_step = TERM_CART_VEL, role, first, last
    t.link, t.target_slot, t.max_displacement = link, -1, max_displacement
    return t


def collision_term(role, first, last, margin, coeff, buffer=0.01, fixed_steps=(), evaluator=COLL_DISCRETE, lvs=0.5):
    t = Term()
    t.kind, t.role, t.first_step, t.last_step = TERM_COLLISION, role, first, last
    t.evaluator_type = evaluator
    t.n_fixed_steps = len(fixed_steps)
    for i, s in enumerate(fixed_steps):
        t.fixed_steps[i] = s
    t.margin, t.coeff, t.margin_buffer, t.longest_valid_segment_length = margin, coeff, buffer, lvs
    return t


def interpolate(q0, q1, T):
    """JOINT_INTERPOLATED init (LinSpaced per joint, problem_description.cpp:351-355)."""
    w = np.linspace(0.0, 1.0, T)[None, :, None]
    return q0[:, None, :] * (1 - w) + q1[:, None, :] * w


def config0():
    """configs[0]: single PR2 arm, 10 waypoints, JointVel cost + JointPos constraint (joint_costs_unit.cpp shapes)."""
    robot = robots.pr2_arm("r", with_spheres=False)
    T, D = 10, 7
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1, coeffs=10.0, targets=0.1),
             joint_term(TERM_JOINT_POS, ROLE_CNT, D, 0, 0, coeffs=10.0, targets=0.0)]
    init = np.zeros((1, T, D))
    return ProblemDesc(robot, T, terms, init)


def _sample_endpoints(rng, robot, B):
    lo, hi = np.array(robot["lower"]), np.array(robot["upper"])
    w = hi - lo
    q0 = rng.uniform(lo + 0.1 * w, hi - 0.1 * w, size=(B, len(lo)))
    q1 = rng.uniform(lo + 0.1 * w, hi - 0.1 * w, size=(B, len(lo)))
    return q0, q1


def _targets_from_goal(robot, q_goal, link):
    out = np.zeros((len(q_goal), 1, 7))
    for b, q in enumerate(q_goal):
        R, p = robots.fk_numpy(robot, q)[link]
        out[b, 0, :3] = p
        out[b, 0, 3:] = robots.rot_to_wxyz(R)
    return out


def config1(B=1024, T=30, seed=SEED + 1):
    """configs[1]: JointVel + JointAcc costs, fixed start, CartPose EQ constraint at the last waypoint
    with target FK(q_goal) (feasible by construction)."""
    robot = robots.pr2_arm("r", with_spheres=False)
    rng = np.random.default_rng(seed)
    D = 7
    q0, q1 = _sample_endpoints(rng, robot, B)
    init = interpolate(q0, q1, T)
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1), joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1),
             cart_pose_term(ROLE_CNT, T - 1, robot["tool"], target_slot=0)]
    return ProblemDesc(robot, T, terms, init, fixed_timesteps=[0], cart_targets=_targets_from_goal(robot, q1, robot["tool"]))


def config2(B=1024, T=30, seed=SEED + 2, n_obstacles=8, obstacle_radius=0.10):
    """configs[2]: configs[1] + discrete collision CONSTRAINT (8 sphere obstacles, dist_pen 0.02, coeff 20,
    buffer 0.01) at all non-fixed steps; per-trajectory worlds rejection-sampled for start/goal clearance 0.05.
    More and larger obstacles make the crowded world of scripts/multi_start.py."""
    robot = robots.pr2_arm("r", with_spheres=True)
    rng = np.random.default_rng(seed)
    D = 7
    q0, q1 = _sample_endpoints(rng, robot, B)
    init = interpolate(q0, q1, T)
    obstacles = _sample_obstacles(rng, robot, q0, q1, n_obstacles, obstacle_radius)
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1), joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1),
             cart_pose_term(ROLE_CNT, T - 1, robot["tool"], target_slot=0),
             collision_term(ROLE_CNT, 0, T - 1, margin=0.02, coeff=20.0, buffer=0.01, fixed_steps=[0])]
    return ProblemDesc(robot, T, terms, init, fixed_timesteps=[0],
                       cart_targets=_targets_from_goal(robot, q1, robot["tool"]), obstacles=obstacles)


def _sample_obstacles(rng, robot, q0, q1, n_obstacles, radius=0.10):
    B = len(q0)
    radii = np.array([s.radius for s in robot["spheres"]])
    obstacles = np.zeros((B, n_obstacles, 4))
    lo, hi = np.array([0.35, -0.70, 0.55]), np.array([0.95, 0.10, 1.25])
    for b in range(B):
        ends = np.concatenate([robots.sphere_centers(robot, q0[b]), robots.sphere_centers(robot, q1[b])])
        rr = np.concatenate([radii, radii])
        k = 0
        while k < n_obstacles:
            c = rng.uniform(lo, hi)
            if np.min(np.linalg.norm(ends - c, axis=1) - rr - radius) >= 0.05:
                obstacles[b, k] = (*c, radius)
                k += 1
    return obstacles


def seed_trajectories(start, goal, T, n_seeds, rng, spread, lower=None, upper=None):
    """Initial trajectories for a multi-start solve: [P * n_seeds, T, D], the n_seeds seeds of problem p at rows
    [p * n_seeds, (p + 1) * n_seeds) (the group layout of tb200_problem_desc.group_size).  Seed 0 is the straight joint
    interpolation start -> goal; seed k > 0 interpolates linearly through a mid waypoint (at (T - 1) // 2) drawn
    uniformly within +-spread of the straight line's midpoint per joint and clamped to [lower, upper].  Endpoints are
    kept exactly.  Deterministic given the state of `rng` (numpy Generator); host-side."""
    start = np.atleast_2d(np.asarray(start, dtype=np.float64))
    goal = np.atleast_2d(np.asarray(goal, dtype=np.float64))
    P, D = start.shape
    straight = interpolate(start, goal, T)
    out = np.repeat(straight, n_seeds, axis=0).reshape(P, n_seeds, T, D)
    m = (T - 1) // 2
    if n_seeds > 1 and m > 0:
        mid = 0.5 * (start + goal)
        off = rng.uniform(-spread, spread, size=(P, n_seeds - 1, D))
        via = mid[:, None, :] + off
        if lower is not None:
            via = np.maximum(via, np.asarray(lower, dtype=np.float64))
        if upper is not None:
            via = np.minimum(via, np.asarray(upper, dtype=np.float64))
        for t in range(1, T - 1):
            if t <= m:
                w = t / m
                a, b = start[:, None, :], via
            else:
                w = (t - m) / (T - 1 - m)
                a, b = via, goal[:, None, :]
            out[:, 1:, t] = a * (1 - w) + b * w
    return out.reshape(P * n_seeds, T, D)


def with_seeds(desc, n_seeds, rng, spread, group_stop=0):
    """The multi-start form of a description: every trajectory becomes a group of n_seeds seeds (seed_trajectories
    between its first and last initial waypoints, clamped to the robot's limits) that share its targets and world."""
    d = desc
    init = seed_trajectories(d.init_traj[:, 0], d.init_traj[:, -1], d.T, n_seeds, rng, spread,
                             d.robot_spec["lower"], d.robot_spec["upper"])
    rep = lambda a: None if a is None else np.repeat(a, n_seeds, axis=0)  # noqa: E731
    per_traj = bool(d.c.obstacles_per_traj)
    return ProblemDesc(d.robot_spec, d.T, d.terms, init, fixed_timesteps=d._fixed_t, fixed_dofs=d._fixed_d,
                       cart_targets=rep(d.cart_targets), obstacles=rep(d.obstacles) if per_traj else d.obstacles,
                       obstacles_per_traj=per_traj, sqp=d.c.sqp, qp=d.c.qp, group_size=n_seeds, group_stop=group_stop,
                       sqp_per_traj=None if d.sqp_per_traj is None else [r for r in d.sqp_per_traj for _ in range(n_seeds)])


def config3(B=4096, T=50, seed=SEED + 3, n_obstacles=8, via_every=10, lvs=0.05, evaluator=COLL_LVS_CONTINUOUS):
    """configs[3]: the configs[2] world with LVS_CONTINUOUS collision (longest_valid_segment_length 0.05) between
    consecutive waypoints, position-only CartPose constraints on every 10th waypoint along the straight Cartesian
    line start -> goal, the full CartPose constraint at the last waypoint, and a CartVel INEQ constraint
    (max_displacement 0.05) on every step pair (SURVEY.md section 8d).  `evaluator=COLL_LVS_DISCRETE` swaps the swept test
    for discrete tests at the interpolated states (DiscreteCollisionEvaluator, collision_terms.cpp:744-893)."""
    robot = robots.pr2_arm("r", with_spheres=True)
    rng = np.random.default_rng(seed)
    D = 7
    q0, q1 = _sample_endpoints(rng, robot, B)
    init = interpolate(q0, q1, T)
    obstacles = _sample_obstacles(rng, robot, q0, q1, n_obstacles)
    tool = robot["tool"]
    goal = _targets_from_goal(robot, q1, tool)[:, 0]
    start = _targets_from_goal(robot, q0, tool)[:, 0]
    vias = [t for t in range(via_every, T - 1, via_every)]
    targets = np.zeros((B, len(vias) + 1, 7))
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1), joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1)]
    for k, t in enumerate(vias):
        w = t / (T - 1)
        targets[:, k, :3] = (1 - w) * start[:, :3] + w * goal[:, :3]
        targets[:, k, 3:] = goal[:, 3:]
        terms.append(cart_pose_term(ROLE_CNT, t, tool, target_slot=k, rot_coeffs=(0, 0, 0)))
    targets[:, len(vias)] = goal
    terms.append(cart_pose_term(ROLE_CNT, T - 1, tool, target_slot=len(vias)))
    terms.append(cart_vel_term(ROLE_CNT, 0, T - 2, tool, 0.05))
    terms.append(collision_term(ROLE_CNT, 0, T - 1, margin=0.02, coeff=20.0, buffer=0.01, fixed_steps=[0],
                                evaluator=evaluator, lvs=lvs))
    return ProblemDesc(robot, T, terms, init, fixed_timesteps=[0], cart_targets=targets, obstacles=obstacles)


def config_variants(B=8, T=10, seed=SEED + 7, n_obstacles=8):
    """Every term flavour the device path has that configs[1]-[3] do not use: JointVel cost with a target, JointAcc
    INEQ cost, JointPos INEQ constraint (a band around the initial path), CartPose as an ABS cost (position only),
    CartVel as an ABS cost, collision as a hinge COST, one fixed DOF (fixed_dofs) on top of the fixed first waypoint."""
    robot = robots.pr2_arm("r", with_spheres=True)
    rng = np.random.default_rng(seed)
    D = 7
    q0, q1 = _sample_endpoints(rng, robot, B)
    init = interpolate(q0, q1, T)
    obstacles = _sample_obstacles(rng, robot, q0, q1, n_obstacles)
    tool = robot["tool"]
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1, coeffs=2.0, targets=0.01),
             joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1, coeffs=1.0, upper=0.05, lower=-0.05),
             cart_pose_term(ROLE_COST, T - 1, tool, target_slot=0, rot_coeffs=(0, 0, 0), pos_coeffs=(5, 5, 5)),
             cart_vel_term(ROLE_COST, 0, T - 2, tool, 0.08),
             collision_term(ROLE_COST, 0, T - 1, margin=0.02, coeff=20.0, buffer=0.01, fixed_steps=[0]),
             joint_term(TERM_JOINT_POS, ROLE_CNT, D, 1, T - 1, coeffs=1.0, upper=[3.2] * 6 + [7.0], lower=[-3.2] * 6 + [-7.0])]
    return ProblemDesc(robot, T, terms, init, fixed_timesteps=[0], fixed_dofs=[6],
                       cart_targets=_targets_from_goal(robot, q1, tool), obstacles=obstacles)


def _rotvec(R):
    """Rotation vector (axis * angle) of a rotation matrix."""
    c = min(1.0, max(-1.0, (np.trace(R) - 1.0) / 2.0))
    ang = np.arccos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    n = np.linalg.norm(w)
    return np.zeros(3) if n < 1e-14 else w / n * ang


def _ik_to_pose(robot, q, link, joints, p_goal, R_goal, iters=200):
    """Host-side damped least squares IK over `joints` (problem generation only: the synthetic goals of configs[4]
    must be reachable).  Returns the joint vector or None."""
    q = q.copy()
    lo, hi = np.array(robot["lower"]), np.array(robot["upper"])
    segs = robot["segments"]
    for _ in range(iters):
        fr = robots.fk_numpy(robot, q)
        R, p = fr[link]
        e = np.concatenate([p_goal - p, _rotvec(R_goal @ R.T)])
        if np.abs(e).max() < 1e-12:
            return q
        J = np.zeros((6, len(joints)))
        anc, a = set(), link
        while a >= 0:
            anc.add(a)
            a = segs[a].parent
        for k, j in enumerate(joints):
            sg = next(i for i, g in enumerate(segs) if g.q_index == j)
            if sg not in anc:
                continue
            Rj, pj = fr[sg]
            ax = Rj @ np.array(list(segs[sg].axis))
            J[:3, k], J[3:, k] = np.cross(ax, p - pj), ax
        dq = J.T @ np.linalg.solve(J @ J.T + 1e-6 * np.eye(6), e)
        step = np.abs(dq).max()
        if step > 0.2:
            dq *= 0.2 / step
        q[joints] = q[joints] + dq
        if (q < lo + 1e-3).any() or (q > hi - 1e-3).any():
            return None
    return None


def config4(B=256, T=40, seed=SEED + 4, n_obstacles=8, trust_box_size=None, trust_shrink_ratio=None,
            trust_expand_ratio=None):
    """configs[4]: 14-DOF dual arm (both PR2 arms on torso_lift_link, tree FK), 40 waypoints, the "glass upright"
    pattern of the reference's README (README.md:57-60): a CartPose constraint with pos_coeffs 0 and rot_coeffs (1,1,0)
    per gripper on every free waypoint (zero coefficients are dropped by hatch, problem_description.cpp:910-926), a full
    CartPose constraint per gripper at the last waypoint, discrete collision constraints (14 robot spheres x 8 obstacle
    spheres) at every free waypoint, JointVel + JointAcc costs, fixed first waypoint, JOINT_INTERPOLATED initial
    trajectory.  The goal of each gripper lies 0.15-0.30 m from its start position and is rotated about the upright axis
    (the target frame's z) only, so that start and goal both satisfy the upright constraint; the goal joint state comes
    from a host-side IK (problem generation), the pose target is FK(q_goal).  The trust-region sweep of SURVEY.md
    section 8d overrides trust_box_size / trust_shrink_ratio / trust_expand_ratio."""
    robot = robots.pr2_dual_arm()
    rng = np.random.default_rng(seed)
    D = 14
    lo_q, hi_q = np.array(robot["lower"]), np.array(robot["upper"])
    w_q = hi_q - lo_q
    tools = (robot["tool"], robot["tool_left"])
    arm_joints = (np.arange(0, 7), np.arange(7, 14))
    q0 = np.zeros((B, D))
    q1 = np.zeros((B, D))
    targets = np.zeros((B, 2, 7))
    radii = np.array([s.radius for s in robot["spheres"]])
    obstacles = np.zeros((B, n_obstacles, 4))
    lo, hi = np.array([0.30, -0.75, 0.50]), np.array([0.95, 0.75, 1.30])
    for b in range(B):
        while True:  # a start state whose two goals are reachable
            qs = rng.uniform(lo_q + 0.2 * w_q, hi_q - 0.2 * w_q)
            fr = robots.fk_numpy(robot, qs)
            qg = qs.copy()
            ok = True
            for a, link in enumerate(tools):
                R, p = fr[link]
                v = rng.standard_normal(3)
                step = v / np.linalg.norm(v) * rng.uniform(0.15, 0.30)
                th = rng.uniform(-0.6, 0.6)
                Rz = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
                sol = _ik_to_pose(robot, qg, link, arm_joints[a], p + step, R @ Rz)
                if sol is None:
                    ok = False
                    break
                qg = sol
            if ok:
                break
        q0[b], q1[b] = qs, qg
        frg = robots.fk_numpy(robot, qg)
        goals = []
        for a, link in enumerate(tools):
            R, p = frg[link]
            targets[b, a, :3] = p
            targets[b, a, 3:] = robots.rot_to_wxyz(R)
            goals.append(p)
        ends = np.concatenate([robots.sphere_centers(robot, qs), robots.sphere_centers(robot, qg)])
        rr = np.concatenate([radii, radii])
        k = 0
        while k < n_obstacles:
            c = rng.uniform(lo, hi)
            if np.min(np.linalg.norm(ends - c, axis=1) - rr - 0.10) >= 0.05:
                obstacles[b, k] = (*c, 0.10)
                k += 1
    init = interpolate(q0, q1, T)
    terms = [joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1), joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1)]
    for t in range(1, T - 1):
        for a, link in enumerate(tools):
            terms.append(cart_pose_term(ROLE_CNT, t, link, target_slot=a, pos_coeffs=(0, 0, 0), rot_coeffs=(1, 1, 0)))
    for a, link in enumerate(tools):
        terms.append(cart_pose_term(ROLE_CNT, T - 1, link, target_slot=a))
    terms.append(collision_term(ROLE_CNT, 0, T - 1, margin=0.02, coeff=20.0, buffer=0.01, fixed_steps=[0]))
    sqp = capi.default_sqp_params()
    if trust_box_size is not None:
        sqp.trust_box_size = trust_box_size
    if trust_shrink_ratio is not None:
        sqp.trust_shrink_ratio = trust_shrink_ratio
    if trust_expand_ratio is not None:
        sqp.trust_expand_ratio = trust_expand_ratio
    return ProblemDesc(robot, T, terms, init, fixed_timesteps=[0], cart_targets=targets, obstacles=obstacles, sqp=sqp)


# the trust-region sweep of configs[4] (SURVEY.md section 8d)
CONFIG4_SWEEP = [(tb, sh, ex) for tb in (0.01, 0.05, 0.1, 0.5) for sh in (0.1, 0.5) for ex in (1.2, 1.5, 2.0)]


def sweep(desc, param_sets):
    """A parameter sweep as one batch: the description tiled once per parameter set (capi.SqpParams), trajectories
    [k*B, (k+1)*B) running under param_sets[k].  Returns the tiled description, whose per-trajectory table holds those
    rows, and the set index of every trajectory ([len(param_sets) * B]).  Groups stay whole: every tile is the whole
    batch."""
    d, K = desc, len(param_sets)
    if K < 1:
        raise ValueError("no parameter sets")
    tile = lambda a: None if a is None else np.concatenate([a] * K, axis=0)  # noqa: E731
    per_traj = bool(d.c.obstacles_per_traj)
    rows = [p for p in param_sets for _ in range(d.B)]
    out = ProblemDesc(d.robot_spec, d.T, d.terms, tile(d.init_traj), fixed_timesteps=d._fixed_t, fixed_dofs=d._fixed_d,
                      cart_targets=tile(d.cart_targets), obstacles=tile(d.obstacles) if per_traj else d.obstacles,
                      obstacles_per_traj=per_traj, sqp=d.c.sqp, qp=d.c.qp, group_size=d.c.group_size,
                      group_stop=d.c.group_stop, sqp_per_traj=rows)
    return out, np.repeat(np.arange(K, dtype=np.int32), d.B)

CONFIGS = {"cfg0": config0, "cfg1": config1, "cfg2": config2, "cfg3": config3, "cfg4": config4, "variants": config_variants}
