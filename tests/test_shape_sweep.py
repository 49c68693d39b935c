"""Shape sweep of the QP step and the kernel instances.

The QP step picks its code path per problem shape and per QP: the ADMM block (admm_block_pinv, admm_block_fast,
admm_block, admm_block_soa), the factor and the objective band in shared or global memory, the rows of the QP in shared
memory or (more than row_cap of them) in global memory, the polish refinement by polish_passes or by the generic
passes.  The convexify and persistent solve kernels come in instances for 2, 3, 6, 7 and 14 joints, with two-waypoint
rows for 2 and 7.  The cases below sit on the switch points of those choices (qp_smem_layout, pinv_plan and
solve_roles_fit of qp_cta_kernel.cuh, which tb200_debug_qp_layout evaluates on the host), and every one of them is
compared with the CPU oracle at the tolerances of test_gpu_parity.py.  The device reports which paths each
trajectory's QPs took (tb200_debug_qp_paths): every case asserts the paths its shape decides, and the whole sweep
asserts that every path was reached, so that a layout change that silently drops a path fails here.  Since every
comparison of a polished QP is blind to the arithmetic of the ADMM blocks (the polish recomputes the minimiser from the
raw rows), one case per block is also compared without polish, on the ADMM iterate itself.

New fixtures: a 6-DOF PR2 arm (forearm roll held FIXED between two moving joints), a 3-DOF revolute-prismatic-revolute
arm whose joint columns are permuted against its segment order, and spherebot (2 DOF) with discrete and with
LVS-continuous collision.  Their discrete collision rows are also checked against plain numpy (FK sphere centres,
central differences), which catches an FK / Jacobian error the oracle and the kernel would share.

The part without a marker runs without a GPU: the oracle solves every case, the new robots' numpy FK agrees with the
oracle's, the numpy collision rows agree with the oracle's, every case passes validation, and the shapes the library
refuses are refused with TB200_ERR_UNSUPPORTED and a message before any device is touched."""
import ctypes as C
import math
import time
import zlib

import numpy as np
import pytest

from trajopt_b200 import api, capi, problems, robots
from trajopt_b200.capi import (COLL_DISCRETE, COLL_LVS_CONTINUOUS, JOINT_FIXED, JOINT_PRISMATIC, JOINT_REVOLUTE,
                               ROLE_CNT, ROLE_COST, TERM_JOINT_ACC, TERM_JOINT_POS, TERM_JOINT_VEL)

# the tolerances of test_gpu_parity.py
ROW_RTOL = 1e-10
QP_X_ATOL = 1e-7
COST_ATOL = 1e-6

# QpPath bits of qp_cta_kernel.cuh
PINV, FAST, GENERIC, SOA = 1 << 0, 1 << 1, 1 << 2, 1 << 3
FACTOR_G, BAND_G, ROWS_G = 1 << 4, 1 << 5, 1 << 6
FUSED, POLISH_FAST, POLISH_GENERIC = 1 << 7, 1 << 8, 1 << 9
PATH_NAMES = [(PINV, "pinv"), (FAST, "fast"), (GENERIC, "block"), (SOA, "soa"), (FACTOR_G, "factor_g"),
              (BAND_G, "band_g"), (ROWS_G, "rows_g"), (FUSED, "fused"), (POLISH_FAST, "pol_fast"),
              (POLISH_GENERIC, "pol_gen")]
BLOCKS = PINV | FAST | GENERIC


# ---------------------------------------------------------------------------------------------------- robots
def pr2_arm_6dof():
    """The PR2 right arm with r_forearm_roll_joint FIXED: a fixed joint between two moving ones, 6 DOF, the 7 spheres
    of the 7-DOF arm (one of them on the now fixed forearm roll link)."""
    r = robots.pr2_arm("r")
    k = r["link_names"].index("r_forearm_roll_link")
    segs = [capi.Segment.from_buffer_copy(s) for s in r["segments"]]
    qk = segs[k].q_index
    segs[k].joint_type, segs[k].q_index = JOINT_FIXED, -1
    for s in segs:
        if s.q_index > qk:
            s.q_index -= 1
    return dict(n_dof=6, segments=segs, lower=r["lower"][:qk] + r["lower"][qk + 1:],
                upper=r["upper"][:qk] + r["upper"][qk + 1:],
                spheres=[capi.Sphere.from_buffer_copy(s) for s in r["spheres"]], link_names=r["link_names"],
                tool=r["tool"])


def rpr_arm():
    """3 DOF: revolute (z) -> prismatic along the link (x) -> revolute (y, in a frame tilted 45 degrees about x), a
    sphere on each link and one at the tool.  The joint columns are permuted: the segments in chain order hold the
    columns 2, 0, 1 (so q[0] is the prismatic joint)."""
    c, s = math.cos(math.pi / 8), math.sin(math.pi / 8)
    segs = [robots._seg(-1, JOINT_FIXED, -1, (0, 0, 0.2)),
            robots._seg(0, JOINT_REVOLUTE, 2, (0, 0, 0.1), (0, 0, 1)),
            robots._seg(1, JOINT_PRISMATIC, 0, (0.25, 0, 0), (1, 0, 0)),
            robots._seg(2, JOINT_REVOLUTE, 1, (0.3, 0, 0), (0, 1, 0), wxyz=(c, s, 0, 0)),
            robots._seg(3, JOINT_FIXED, -1, (0.25, 0, 0))]
    spheres = [robots._sphere(1, (0.12, 0, 0), 0.08), robots._sphere(2, (0.15, 0, 0), 0.07),
               robots._sphere(3, (0.12, 0, 0), 0.06), robots._sphere(4, (0, 0, 0), 0.05)]
    return dict(n_dof=3, segments=segs, lower=[0.0, -1.5, -2.5], upper=[0.3, 1.5, 2.5], spheres=spheres,
                link_names=["base", "link1", "link2", "link3", "tool"], tool=4)


ROBOTS = {2: robots.spherebot, 3: rpr_arm, 6: pr2_arm_6dof, 7: lambda: robots.pr2_arm("r"), 14: robots.pr2_dual_arm}


def _endpoints(rng, robot, B):
    if robot["n_dof"] == 2:  # spherebot: +-20 m limits; moves of a few sphere diameters
        q0 = rng.uniform(-1.5, 1.5, size=(B, 2))
        return q0, q0 + rng.uniform(-1.5, 1.5, size=(B, 2))
    lo, hi = np.array(robot["lower"]), np.array(robot["upper"])
    w = hi - lo
    return (rng.uniform(lo + 0.1 * w, hi - 0.1 * w, size=(B, len(lo))),
            rng.uniform(lo + 0.1 * w, hi - 0.1 * w, size=(B, len(lo))))


def _obstacles(rng, robot, q0, q1, n, shared):
    """n obstacle spheres per trajectory (one world for the batch when `shared`) in the box of the robot spheres
    along the straight joint path, 0.05 clear of every robot sphere at start and goal."""
    r_obs = 0.3 if robot["n_dof"] == 2 else 0.1
    radii = np.array([s.radius for s in robot["spheres"]])
    worlds = [np.arange(len(q0))] if shared else [[b] for b in range(len(q0))]
    out = np.zeros((len(worlds), n, 4))
    for k, members in enumerate(worlds):
        path = np.concatenate([robots.sphere_centers(robot, (1 - w) * q0[b] + w * q1[b])
                               for b in members for w in np.linspace(0, 1, 5)])
        ends = np.concatenate([robots.sphere_centers(robot, q) for b in members for q in (q0[b], q1[b])])
        rr = np.tile(radii, len(ends) // len(radii))
        pad = np.array([1.0, 1.0, 0.2]) if robot["n_dof"] == 2 else 0.2  # (spherebot moves in the plane z = 0)
        lo, hi = path.min(0) - pad, path.max(0) + pad
        m = 0
        for _ in range(200000):
            c = rng.uniform(lo, hi)
            if np.min(np.linalg.norm(ends - c, axis=1) - rr - r_obs) >= 0.05:
                out[k, m] = (*c, r_obs)
                m += 1
                if m == n:
                    break
        assert m == n, "obstacle sampling did not fill the world"
    return out


def build_case(D, T, B=4, pair=False, n_obstacles=8, buffer=0.01, shared=False, seed=0):
    """The configs[2] / configs[3] term mix on any robot: JointVel + JointAcc costs, a CartPose constraint at the last
    waypoint (position only for <= 3 DOF; x, y for spherebot) with target FK(q_goal), collision constraints on every
    free waypoint (discrete; LVS-continuous with `pair`) and with `pair` a CartVel constraint on every step pair.  Terms
    the length cannot hold are dropped: T = 1 is a JointPos cost alone, T = 2 has no JointAcc."""
    robot = ROBOTS[D]()
    rng = np.random.default_rng(seed)
    q0, q1 = _endpoints(rng, robot, B)
    init = problems.interpolate(q0, q1, T)
    if T == 1:
        mid = 0.5 * (np.array(robot["lower"]) + np.array(robot["upper"]))
        terms = [problems.joint_term(TERM_JOINT_POS, ROLE_COST, D, 0, 0, coeffs=2.0, targets=mid)]
        return capi.ProblemDesc(robot, T, terms, init)
    tool = robot["tool"]
    terms = [problems.joint_term(TERM_JOINT_VEL, ROLE_COST, D, 0, T - 1)]
    if T >= 3:
        terms.append(problems.joint_term(TERM_JOINT_ACC, ROLE_COST, D, 0, T - 1))
    pos = (1, 1, 0) if D == 2 else (1, 1, 1)
    rot = (0, 0, 0) if D <= 3 else (1, 1, 1)
    terms.append(problems.cart_pose_term(ROLE_CNT, T - 1, tool, target_slot=0, pos_coeffs=pos, rot_coeffs=rot))
    if pair:  # a step limit the length can meet (configs[3]: 0.05 at 50 waypoints)
        max_disp = max(0.3, 3.0 / (T - 1)) if D == 2 else max(0.05, 2.5 / (T - 1))
        terms.append(problems.cart_vel_term(ROLE_CNT, 0, T - 2, tool, max_disp))
    terms.append(problems.collision_term(ROLE_CNT, 0, T - 1, margin=0.02, coeff=20.0, buffer=buffer, fixed_steps=[0],
                                         evaluator=COLL_LVS_CONTINUOUS if pair else COLL_DISCRETE,
                                         lvs=0.5 if D == 2 else 0.1))
    obstacles = _obstacles(rng, robot, q0, q1, n_obstacles, shared)
    return capi.ProblemDesc(robot, T, terms, init, fixed_timesteps=[0],
                            cart_targets=problems._targets_from_goal(robot, q1, tool), obstacles=obstacles,
                            obstacles_per_traj=not shared)


# ---------------------------------------------------------------------------------------------------- the sweep
def _cases():
    c = {}
    for T in (1, 3, 5, 7, 15, 16, 23, 24, 25, 27, 31, 33, 36, 37, 49, 59, 64):
        c[f"d7_T{T}"] = dict(D=7, T=T)
    # (continuous collision: B = 8, for the share of trajectories test_sqp_solve_matches_oracle compares step by step)
    for T in (5, 16, 24, 33, 64):
        c[f"d7p_T{T}"] = dict(D=7, T=T, pair=True, B=8)
    # (6 joints at 64 waypoints, seed of "d6_T64", is not a case: trajectory 1 converges one QP earlier than the oracle
    # after 15 QPs, each ending in a KKT-verified polish with model merits equal to 5e-11, because its 15th step meets
    # the min_approx_improve test at 0.992e-4 against 1.019e-4 in the oracle - a 1e-4 threshold that the 1e-10
    # differences of the two back ends, grown over 14 accepted steps, cross.  41 waypoints take the same block.)
    for D, Ts in ((6, (3, 9, 16, 24, 33, 41)), (3, (3, 9, 16, 24, 33, 64))):
        for T in Ts:
            c[f"d{D}_T{T}"] = dict(D=D, T=T)
    for T in (2, 13, 40):
        # (24 obstacles with a 0.1 buffer: a spherebot world with contacts at most waypoints)
        c[f"d2_T{T}"] = dict(D=2, T=T, n_obstacles=24, buffer=0.1)
        c[f"d2p_T{T}"] = dict(D=2, T=T, pair=True, B=8)
    for T in (3, 9, 17, 50, 62):  # (64 waypoints of 14 joints are refused: test_unsupported_shape_is_refused)
        c[f"d14_T{T}"] = dict(D=14, T=T)
    # crowded worlds: more rows than row_cap at partition-inverse sizes (admm_block_soa), masks of several words
    c["d7_T12_crowded"] = dict(D=7, T=12, n_obstacles=40, buffer=0.3)
    c["d7_T10_obs64"] = dict(D=7, T=10, n_obstacles=64)
    c["d7_T10_obs64_shared"] = dict(D=7, T=10, n_obstacles=64, shared=True)
    return c


CASES = _cases()
NEW_ROBOT_DISCRETE = [k for k, v in CASES.items() if v["D"] in (2, 3, 6) and not v.get("pair") and v["T"] >= 2]


class _Descs(dict):
    def __missing__(self, name):
        self[name] = build_case(seed=zlib.crc32(name.encode()), **CASES[name])
        return self[name]


DESCS = _Descs()


# ---------------------------------------------------------------------------------------------------- layout model
def predict_layout(desc, L):
    """What the shape decides (tb200_debug_qp_layout: qp_smem_layout and qp_plan of qp_cta_kernel.cuh on the host):
    the ADMM block of a QP whose rows fit shared memory, factor / band in global memory, row_cap and max_rows (rows
    beyond row_cap go to global memory and through admm_block_soa), the polish variant."""
    D = desc.D
    pair = L.coll_row_stride == 2 * D + 3 or L.cart_jac_stride == 2 * D
    max_rows = max(1, len(desc._fixed_t) * D + L.n_cart_rows + L.n_coll_cand)
    out = np.zeros(8, np.int32)
    lib = capi.load_library()
    assert lib.tb200_debug_qp_layout(desc.T, D, int(pair), max_rows, out.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    return dict(M=int(out[0]), factor_g=bool(out[1]), band_g=bool(out[2]), row_cap=int(out[3]), block=int(out[4]),
                fused=bool(out[5]), fast_polish=bool(out[6]), max_rows=max_rows)


def _check_paths(name, desc, L, bits, generic_passes=False):
    """The paths of one run (per trajectory) against what the shape decides."""
    pr = predict_layout(desc, L)
    for b, v in enumerate(bits):
        v = int(v)
        msg = (name, b, _names(v), pr)
        assert bool(v & FACTOR_G) == pr["factor_g"], msg
        assert bool(v & BAND_G) == pr["band_g"], msg
        assert bool(v & ROWS_G) == bool(v & SOA), msg  # rows in global memory <=> admm_block_soa
        if pr["max_rows"] <= pr["row_cap"]:
            assert not v & ROWS_G, msg
        # the block of QPs with their rows on chip is the one the shape decides; all QPs spilled: none of them
        assert v & BLOCKS in ((pr["block"], 0) if v & ROWS_G else (pr["block"],)), msg
        if not v & PINV or generic_passes:
            assert not v & (FUSED | POLISH_FAST), msg
        if v & POLISH_FAST:
            assert pr["fast_polish"], msg
        if v & PINV and not generic_passes and v & (POLISH_FAST | POLISH_GENERIC) and not v & ROWS_G:
            assert v & (POLISH_FAST if pr["fast_polish"] else POLISH_GENERIC), msg
    return pr


def _names(v):
    return "|".join(n for bit, n in PATH_NAMES if v & bit) or "-"


# ---------------------------------------------------------------------------------------------------- numpy reference
def _dist_fn(robot, s, ob):
    sp = robot["spheres"][s]
    cen = np.array(list(sp.center))

    def f(q):
        R, p = robots.fk_numpy(robot, q)[sp.segment]
        return np.linalg.norm(R @ cen + p - ob[:3]) - sp.radius - ob[3]
    return f


def check_coll_rows_numpy(desc, x, rows):
    """Discrete collision rows [gradient(D), dist, margin, coeff or 0] in the oracle's candidate order (free waypoint,
    robot sphere, obstacle) against plain numpy: dist0 = |c_s(q) - c_o| - r_s - r_o from fk_numpy, the gradient against
    central differences (h = 1e-6) of that distance, active = dist0 <= margin + buffer (inactive rows: zero gradient)."""
    robot, D = desc.robot_spec, desc.D
    term = next(t for t in desc.terms if t.kind == capi.TERM_COLLISION)
    fixed = set(term.fixed_steps[:term.n_fixed_steps])
    steps = [t for t in range(term.first_step, term.last_step + 1) if t not in fixed]
    h = 1e-6
    n_active = 0
    for b in range(desc.B):
        obs = desc.obstacles[b] if desc.c.obstacles_per_traj else desc.obstacles[0]
        k = 0
        for t in steps:
            q = x[b, t]
            for s in range(len(robot["spheres"])):
                for ob in obs:
                    f = _dist_fn(robot, s, ob)
                    d0 = f(q)
                    row = rows[b, k]
                    active = d0 <= term.margin + term.margin_buffer
                    np.testing.assert_allclose(row[D], d0, rtol=1e-12, atol=1e-12, err_msg=str((b, t, s)))
                    assert row[D + 1] == term.margin
                    assert (row[D + 2] != 0) == active, (b, t, s, d0, row)
                    if active:
                        n_active += 1
                        g = np.array([(f(q + h * e) - f(q - h * e)) / (2 * h) for e in np.eye(D)])
                        np.testing.assert_allclose(row[:D], g, rtol=0, atol=1e-7, err_msg=str((b, t, s)))
                        assert row[D + 2] == term.coeff
                    else:
                        assert (row[:D] == 0).all()
                    k += 1
    assert k == rows.shape[1]
    return n_active


def _probe_x(desc):
    rng = np.random.default_rng(7)
    return desc.init_traj + 0.05 * rng.standard_normal(desc.init_traj.shape)


# ====================================================================================================== CPU part
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


@pytest.mark.parametrize("name", list(CASES))
def test_case_passes_validation(name):
    rc, msg = _create(DESCS[name])
    assert rc == (capi.ERR_NO_DEVICE if _no_device() else capi.OK), (rc, msg)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_solves_case(oracle, name):
    d = DESCS[name]
    ref = oracle.solve_batch(d)
    assert (ref["status"] != capi.OPT_INVALID).all(), ref["status"]
    assert np.isfinite(ref["x"]).all() and np.isfinite(ref["total_cost"]).all()


def test_sweep_reaches_every_layout():
    """The sweep is built to reach every ADMM block, the band and the factor in global memory, more rows than row_cap
    (somewhere) and both polish variants, according to the layout model."""
    from oracle_lib import layout
    seen = 0
    for name in CASES:
        d = DESCS[name]
        pr = predict_layout(d, layout(d))
        seen |= pr["block"] | (FACTOR_G if pr["factor_g"] else 0) | (BAND_G if pr["band_g"] else 0)
        seen |= ROWS_G if pr["max_rows"] > pr["row_cap"] else 0
        seen |= POLISH_FAST if pr["fast_polish"] else POLISH_GENERIC
    assert seen == BLOCKS | FACTOR_G | BAND_G | ROWS_G | POLISH_FAST | POLISH_GENERIC, _names(seen)
    # the switch points of DESIGN.md's fall-back: 16-18 blocks of 14 (31-36 waypoints at 7 joints) leave the partition
    # form for admm_block_fast; 64 waypoints at 7 joints keep the band in global memory
    assert predict_layout(DESCS["d7_T33"], layout(DESCS["d7_T33"]))["block"] == FAST
    assert predict_layout(DESCS["d7_T64"], layout(DESCS["d7_T64"]))["band_g"]
    assert predict_layout(DESCS["d7_T16"], layout(DESCS["d7_T16"]))["block"] == PINV


def _analytic_jacobian(robot, q, link, point):
    """Geometric Jacobian from fk_numpy's frames: column q_index of every moving ancestor of `link`."""
    fr = robots.fk_numpy(robot, q)
    J = np.zeros((6, robot["n_dof"]))
    a = link
    while a >= 0:
        s = robot["segments"][a]
        if s.joint_type != JOINT_FIXED:
            R, p = fr[a]
            ax = R @ np.array(list(s.axis))
            if s.joint_type == JOINT_REVOLUTE:
                J[:3, s.q_index], J[3:, s.q_index] = np.cross(ax, point - p), ax
            else:
                J[:3, s.q_index] = ax
        a = s.parent
    return J


@pytest.mark.parametrize("D", [6, 3, 2])
def test_new_robot_fk_matches_oracle(oracle, D):
    robot = ROBOTS[D]()
    d = capi.ProblemDesc(robot, 1, [], np.zeros((1, 1, D)))
    rng = np.random.default_rng(11 + D)
    lo, hi = np.array(robot["lower"]), np.array(robot["upper"])
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    for _ in range(5):
        q = rng.uniform(np.maximum(lo, -3), np.minimum(hi, 3))
        fr = np.zeros((len(robot["segments"]), 12))
        assert oracle.lib().oracle_fk(C.byref(d.c.robot), dp(q), dp(fr)) == 0
        for k, (R, p) in enumerate(robots.fk_numpy(robot, q)):
            np.testing.assert_allclose(fr[k, :9].reshape(3, 3), R, rtol=0, atol=1e-12)
            np.testing.assert_allclose(fr[k, 9:], p, rtol=0, atol=1e-12)
        # the tool frame and every sphere centre (the points the collision gradient is taken at)
        fk = robots.fk_numpy(robot, q)
        pts = [(robot["tool"], fk[robot["tool"]][1])]
        pts += [(s.segment, fk[s.segment][0] @ np.array(list(s.center)) + fk[s.segment][1]) for s in robot["spheres"]]
        for link, pt in pts:
            J = np.zeros((6, D))
            assert oracle.lib().oracle_jacobian(C.byref(d.c.robot), dp(q), link, dp(np.ascontiguousarray(pt)), dp(J)) == 0
            np.testing.assert_allclose(J, _analytic_jacobian(robot, q, link, pt), rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", NEW_ROBOT_DISCRETE)
def test_numpy_collision_rows_match_oracle(oracle, name):
    d = DESCS[name]
    x = _probe_x(d)
    ref = oracle.convexify_batch(d, x)
    assert check_coll_rows_numpy(d, x, ref["coll_rows"]) > 0 or d.T <= 3  # (short worlds may have no contact)


def _refused():
    """Shapes the library refuses, each with its reason: the message it must come with."""
    def d3_pair():  # CartVel rows span two waypoints: no 3-joint instance has such rows
        return build_case(3, 8, B=1, pair=True, seed=1)

    def obstacles_65():  # the candidate masks of the convexify kernel hold at most 64 obstacles per robot sphere
        return build_case(7, 8, B=1, n_obstacles=65, seed=2)

    def d6_pair():
        return build_case(6, 8, B=1, pair=True, seed=3)

    def eval_smem():  # 14 joints x 64 waypoints (the sweep's 14-joint case stops at 62): the convexify kernel's
        return build_case(14, 64, B=1, seed=4)  # per-waypoint tables exceed the 227 KB of one CTA
    return [("d3_pair", d3_pair, "no kernel instance with two-waypoint rows"),
            ("d6_pair", d6_pair, "no kernel instance with two-waypoint rows"),
            ("obstacles_65", obstacles_65, "more than 64 obstacle spheres"),
            ("eval_smem", eval_smem, "does not fit the 227 KB shared memory")]


@pytest.mark.parametrize("name,make,text", _refused(), ids=[r[0] for r in _refused()])
def test_unsupported_shape_is_refused(name, make, text):
    rc, msg = _create(make())
    assert rc == capi.ERR_UNSUPPORTED and text in msg, (rc, msg)


# ====================================================================================================== GPU part
CENSUS = {}  # case -> OR of the path bits of every QP of every run


def _run(desc, fn, monkeypatch=None, generic=None):
    """Create a problem (TB200_GENERIC_QP_PASSES = generic when given), record the QP paths, run fn(problem); returns
    (fn's result, per-trajectory path bits)."""
    if generic is not None:
        monkeypatch.setenv("TB200_GENERIC_QP_PASSES", generic)
    p = api.Problem(desc)
    try:
        assert p.lib.tb200_debug_enable_qp_paths(p.handle, 1) == 0
        out = fn(p)
        bits = np.zeros(desc.B, np.int32)
        assert p.lib.tb200_debug_qp_paths(p.handle, bits.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    finally:
        p.close()
    return out, bits


def _note(name, bits):
    CENSUS[name] = CENSUS.get(name, 0) | int(np.bitwise_or.reduce(bits))


def _solve_traced(p, cap=600):
    """Solve with the decision trace on; per trajectory, whether one of its QPs ended WITHOUT a KKT-verified polished
    point (the rule of test_gpu_parity._solve_with_trace)."""
    d = p.desc
    assert p.lib.tb200_debug_enable_trace(p.handle, cap) == 0
    got = p.solve()
    tr = np.zeros((d.B, cap, 14))
    tl = np.zeros(d.B, np.int32)
    p.lib.tb200_debug_fetch_trace(p.handle, tr.ctypes.data_as(C.POINTER(C.c_double)), tl.ctypes.data_as(C.POINTER(C.c_int32)))
    got["hit"] = np.array([(tr[b, :tl[b], 7] >= d.c.qp.max_iter).any() or (tr[b, :tl[b], 12] != 1).any()
                           for b in range(d.B)])
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_convexify_rows_match_oracle(oracle, name):
    d = DESCS[name]
    x = _probe_x(d)
    p = api.Problem(d)
    try:
        got = p.convexify(x)
    finally:
        p.close()
    ref = oracle.convexify_batch(d, x)
    np.testing.assert_allclose(got["cart_err"], ref["cart_err"], rtol=ROW_RTOL, atol=1e-12)
    np.testing.assert_allclose(got["cart_jac"], ref["cart_jac"], rtol=1e-6, atol=2e-9)  # FD quotient (test_gpu_parity)
    np.testing.assert_allclose(got["cost_vals"], ref["cost_vals"], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(got["cnt_viols"], ref["cnt_viols"], rtol=1e-9, atol=1e-12)
    if got["coll_rows"].size:
        np.testing.assert_allclose(got["coll_rows"], ref["coll_rows"], rtol=ROW_RTOL, atol=1e-12)
        assert ((got["coll_rows"][..., -1] != 0) == (ref["coll_rows"][..., -1] != 0)).all()
    if name in NEW_ROBOT_DISCRETE:  # and against numpy directly
        assert check_coll_rows_numpy(d, x, got["coll_rows"]) > 0 or d.T <= 3


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("trust", [0.1, 0.01])
def test_qp_solve_matches_oracle(oracle, name, trust):
    d = DESCS[name]
    x = d.init_traj.copy()
    got, bits = _run(d, lambda p: p.qp_solve(x, trust, 10.0))
    _note(name, bits)
    _check_paths(name, d, oracle.layout(d), bits)
    ref = oracle.qp_solve_batch(d, x, trust, 10.0)
    assert (got["qp_status"] == ref["qp_status"]).all()
    assert (got["polish"] == ref["polish"]).all(), (got["polish"], ref["polish"])
    np.testing.assert_allclose(got["new_x"], ref["new_x"], atol=QP_X_ATOL)
    np.testing.assert_allclose(got["model_cnt_viols"], ref["model_cnt_viols"], atol=1e-6)
    np.testing.assert_allclose(got["model_cost_vals"], ref["model_cost_vals"], rtol=1e-6, atol=1e-7)
    # ADMM iteration counts: the diagnostic rule of test_gpu_parity
    assert (got["admm_iters"] == ref["admm_iters"]).mean() >= 0.5, (got["admm_iters"], ref["admm_iters"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sqp_solve_matches_oracle(oracle, name):
    d = DESCS[name]
    got, bits = _run(d, _solve_traced)
    _note(name, bits)
    _check_paths(name, d, oracle.layout(d), bits)
    ref = oracle.solve_batch(d)
    hit = got["hit"]
    # the rules of test_gpu_parity.test_sqp_solve_matches_oracle: continuous collision (two-waypoint rows) is compared
    # step by step only on trajectories whose QPs all ended in a KKT-verified polished point, and strictly where the
    # oracle converged; every other case compares every trajectory
    loose = bool(CASES[name].get("pair"))
    ok = ~hit if loose else np.ones(d.B, bool)
    assert ok.mean() >= 0.75, ("trajectories with an unverified QP", np.nonzero(hit)[0])
    assert (got["status"][ok] == ref["status"][ok]).all(), (got["status"], ref["status"], hit)
    assert (got["n_qp_solves"][ok] == ref["n_qp_solves"][ok]).all(), (got["n_qp_solves"], ref["n_qp_solves"], hit)
    strict = ok & (ref["status"] == capi.OPT_CONVERGED) if loose else ok
    assert strict.any()
    np.testing.assert_allclose(got["total_cost"][strict], ref["total_cost"][strict], atol=COST_ATOL)
    np.testing.assert_allclose(got["x"][strict], ref["x"][strict], atol=1e-5)
    np.testing.assert_allclose(got["cnt_viols"][strict], ref["cnt_viols"][strict], atol=1e-6)
    # (atol: a single waypoint's JointPos cost converges to a rounding of zero, 1e-32 against 1e-31; the strict
    # comparison above already holds every such trajectory to 1e-6)
    np.testing.assert_allclose(got["total_cost"][ok], ref["total_cost"][ok], rtol=5e-3, atol=1e-20)
    assert (got["status"] != capi.OPT_INVALID).all()


# One case of every ADMM block, of a padded last block (odd T at an odd number of joints), of the band and the factor in
# global memory, and of rows spilled at a partition-inverse size.
UNPOLISHED = ["d7_T15", "d7_T16", "d7_T33", "d7_T37", "d7_T59", "d7_T12_crowded", "d7p_T5", "d6_T9", "d3_T33", "d2_T13",
              "d14_T9"]
UNPOLISHED_X_ATOL = 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("name", UNPOLISHED)
def test_admm_iterate_matches_oracle_without_polish(oracle, name):
    """The ADMM iterate itself, not the polished point: without polish and with tolerances of zero, both sides run
    exactly 200 iterations at a fixed rho (adaptive rho off, so that no borderline rho update can separate them) and
    stop at the iteration limit.  The polish of the other tests recomputes the minimiser from the raw rows on the active
    set, so an error in the arithmetic of an ADMM block that leaves the active set alone is invisible there; here it
    moves x.  UNPOLISHED_X_ATOL: 200 iterations of the same map from the same rows, different summation orders."""
    d0 = DESCS[name]
    qp = capi.default_qp_settings()
    qp.polishing, qp.adaptive_rho, qp.early_polish_every, qp.early_polish_from = 0, 0, 0, 0
    qp.eps_abs = qp.eps_rel = qp.eps_prim_inf = qp.eps_dual_inf = 0.0
    qp.max_iter = 200
    d = capi.ProblemDesc(d0.robot_spec, d0.T, d0.terms, d0.init_traj, fixed_timesteps=d0._fixed_t,
                         cart_targets=d0.cart_targets, obstacles=d0.obstacles,
                         obstacles_per_traj=bool(d0.c.obstacles_per_traj), sqp=d0.c.sqp, qp=qp)
    x = d.init_traj.copy()
    got, bits = _run(d, lambda p: p.qp_solve(x, 0.1, 10.0))
    _check_paths(name, d, oracle.layout(d), bits)
    ref = oracle.qp_solve_batch(d, x, 0.1, 10.0)
    print(f"\n{name}: ADMM iterate max|dx| {np.abs(got['new_x'] - ref['new_x']).max():.3e}  paths "
          f"{_names(int(np.bitwise_or.reduce(bits)))}")
    assert (got["admm_iters"] == 200).all() and (ref["admm_iters"] == 200).all(), (got["admm_iters"], ref["admm_iters"])
    assert (got["qp_status"] == ref["qp_status"]).all()
    assert (got["polish"] == 0).all() and (ref["polish"] == 0).all()
    np.testing.assert_allclose(got["new_x"], ref["new_x"], rtol=0, atol=UNPOLISHED_X_ATOL)
    np.testing.assert_allclose(got["model_cnt_viols"], ref["model_cnt_viols"], rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(got["model_cost_vals"], ref["model_cost_vals"], rtol=1e-8, atol=1e-9)


PINV_CASES = [k for k in CASES if CASES[k]["D"] <= 7]  # (filtered to the partition-inverse layouts in the test)


@pytest.mark.gpu
@pytest.mark.parametrize("name", PINV_CASES)
def test_fast_passes_match_generic(oracle, monkeypatch, name):
    """Where the partition-inverse block ran, the fused check and polish_passes against the generic passes
    (TB200_GENERIC_QP_PASSES=1): identical decisions, x within 1e-9 (the pattern of test_fused_check.py)."""
    d = DESCS[name]
    L = oracle.layout(d)
    if predict_layout(d, L)["block"] != PINV:
        pytest.skip("the shape does not take the partition-inverse form")
    x = d.init_traj.copy()
    (gen, gbits), (fus, fbits) = [_run(d, lambda p: p.qp_solve(x, 0.1, 10.0), monkeypatch, g) for g in ("1", "0")]
    _check_paths(name, d, L, gbits, generic_passes=True)
    _check_paths(name, d, L, fbits)
    assert (gen["qp_status"] == fus["qp_status"]).all()
    assert (gen["admm_iters"] == fus["admm_iters"]).all(), (gen["admm_iters"], fus["admm_iters"])
    assert (gen["polish"] == fus["polish"]).all()
    np.testing.assert_allclose(fus["new_x"], gen["new_x"], rtol=0, atol=1e-9)
    (gen, gbits), (fus, fbits) = [_run(d, lambda p: p.solve(), monkeypatch, g) for g in ("1", "0")]
    _check_paths(name, d, L, gbits, generic_passes=True)
    _check_paths(name, d, L, fbits)
    _note(name, fbits)
    for k in ("status", "n_qp_solves", "n_admm_iters"):
        assert (gen[k] == fus[k]).all(), (k, gen[k], fus[k])
    np.testing.assert_allclose(fus["x"], gen["x"], rtol=0, atol=1e-9)
    v = int(np.bitwise_or.reduce(fbits))
    # (crowded worlds: every QP may have spilled its rows to global memory, and then none took the partition form)
    assert v & FUSED or not v & PINV, _names(v)


@pytest.mark.gpu
def test_census_reaches_every_path(oracle):
    """Over the whole sweep every ADMM block, the factor, the band and the rows in global memory, the fused check and
    both polish variants were taken (cases the run before did not cover are solved here)."""
    t0 = time.time()
    for name in CASES:
        if name not in CENSUS:
            d = DESCS[name]
            _, bits = _run(d, lambda p: p.solve())
            _check_paths(name, d, oracle.layout(d), bits)
            _note(name, bits)
    print(f"\nQP path census ({time.time() - t0:.1f} s to complete it)")
    print(f"{'case':<22}{'T':>4}{'D':>4}  paths")
    total = 0
    for name, v in CENSUS.items():
        total |= v
        print(f"{name:<22}{CASES[name]['T']:>4}{CASES[name]['D']:>4}  {_names(v)}")
    print(f"{'(all)':<30}  {_names(total)}")
    for bit, n in PATH_NAMES:
        assert total & bit, f"no case of the sweep reached {n}"
    # rows spilled to global memory at a partition-inverse size (not only by long or wide problems)
    crowded = DESCS["d7_T12_crowded"]
    assert predict_layout(crowded, oracle.layout(crowded))["block"] == PINV
    assert CENSUS["d7_T12_crowded"] & (SOA | ROWS_G) == SOA | ROWS_G, _names(CENSUS["d7_T12_crowded"])
