"""Robot fixtures as tb200_robot descriptions.

Kinematic constants come from the reference's URDF fixtures
(trajopt_common/data/arm_around_table.urdf, spherebot.urdf; groups from pr2.srdf:12-17); they are
data, extracted with tests/golden/extract_urdf.py.  Collision spheres are synthetic (SURVEY.md §8d).
"""
import math

import numpy as np

from .capi import JOINT_FIXED, JOINT_PRISMATIC, JOINT_REVOLUTE, Segment, Sphere


def _seg(parent, jtype, qidx, xyz, axis=(0, 0, 1), wxyz=(1, 0, 0, 0)):
    s = Segment()
    s.parent, s.joint_type, s.q_index = parent, jtype, qidx
    s.origin_xyz[:] = xyz
    s.origin_wxyz[:] = wxyz
    s.axis[:] = axis
    return s


def _sphere(seg, center, radius):
    s = Sphere()
    s.segment = seg
    s.center[:] = center
    s.radius = radius
    return s


# (name, type, origin xyz, axis, lower, upper) along base_footprint -> r_gripper_tool_frame
_PR2_RIGHT = [
    ("base_footprint_joint", JOINT_FIXED, (0, 0, 0.051), None, None, None),
    ("torso_lift_joint", JOINT_FIXED, (-0.05, 0, 0.739675), None, None, None),  # prismatic, held at 0 (planning_unit.cpp:56)
    ("r_shoulder_pan_joint", JOINT_REVOLUTE, (0.0, -0.188, 0.0), (0, 0, 1), -2.2853981634, 0.714601836603),
    ("r_shoulder_lift_joint", JOINT_REVOLUTE, (0.1, 0, 0), (0, 1, 0), -0.5236, 1.3963),
    ("r_upper_arm_roll_joint", JOINT_REVOLUTE, (0, 0, 0), (1, 0, 0), -3.9, 0.8),
    ("r_elbow_flex_joint", JOINT_REVOLUTE, (0.4, 0, 0), (0, 1, 0), -2.3213, 0.0),
    ("r_forearm_roll_joint", JOINT_REVOLUTE, (0, 0, 0), (1, 0, 0), None, None),  # continuous
    ("r_wrist_flex_joint", JOINT_REVOLUTE, (0.321, 0, 0), (0, 1, 0), -2.18, 0.0),
    ("r_wrist_roll_joint", JOINT_REVOLUTE, (0, 0, 0), (1, 0, 0), None, None),  # continuous
    ("r_gripper_tool_joint", JOINT_FIXED, (0.18, 0, 0), None, None, None),
]
_SPHERE_RADII = [0.12, 0.10, 0.09, 0.09, 0.07, 0.06, 0.05]  # SURVEY.md §8d


def _pr2_arm(side, continuous_limit, parent_offset=0, q_offset=0, shared_base=None):
    """Segments of one PR2 arm; side = 'r' or 'l' (left arm mirrored at y=+0.188 with mirrored limits)."""
    segs, lower, upper, names = [], [], [], []
    parent = -1
    q = q_offset
    chain = _PR2_RIGHT
    if shared_base is not None:
        chain = chain[2:]
        parent = shared_base
    for name, jtype, xyz, axis, lo, hi in chain:
        xyz = list(xyz)
        if side == "l":
            name = "l" + name[1:] if name.startswith("r_") else name
            if "shoulder_pan" in name:
                xyz[1] = 0.188
                lo, hi = -hi, -lo
            if "upper_arm_roll" in name:
                lo, hi = -hi, -lo
        qi = -1
        if jtype != JOINT_FIXED:
            qi = q
            q += 1
            if lo is None:
                lo, hi = -continuous_limit, continuous_limit
            lower.append(lo)
            upper.append(hi)
        segs.append(_seg(parent, jtype, qi, xyz, axis or (0, 0, 1)))
        names.append(name.replace("_joint", "_link") if "tool" not in name else side + "_gripper_tool_frame")
        parent = parent_offset + len(segs) - 1
    return segs, lower, upper, names


def pr2_arm(side="r", continuous_limit=2 * math.pi, with_spheres=True):
    """7-DOF PR2 arm rooted at base_footprint (tesseract assigns +-4pi to continuous joints [EXT];
    synthetic runs use +-2pi, SURVEY.md §8d)."""
    segs, lower, upper, names = _pr2_arm(side, continuous_limit)
    spheres = []
    if with_spheres:
        moving = [i for i, s in enumerate(segs) if s.joint_type != JOINT_FIXED]
        at = moving[:-1] + [len(segs) - 1]  # one per moving link frame origin, the last at the tool frame
        spheres = [_sphere(seg, (0, 0, 0), r) for seg, r in zip(at, _SPHERE_RADII)]
    return dict(n_dof=7, segments=segs, lower=lower, upper=upper, spheres=spheres, link_names=names,
                tool=len(segs) - 1)


def pr2_dual_arm(continuous_limit=2 * math.pi):
    """14-DOF tree: both arms hang off torso_lift_link (configs[4]; synthetic group, SURVEY.md §8d)."""
    base = [_seg(-1, JOINT_FIXED, -1, (0, 0, 0.051)), _seg(0, JOINT_FIXED, -1, (-0.05, 0, 0.739675))]
    rs, rl, ru, rn = _pr2_arm("r", continuous_limit, parent_offset=2, q_offset=0, shared_base=1)
    ls, ll, lu, ln = _pr2_arm("l", continuous_limit, parent_offset=2 + len(rs), q_offset=7, shared_base=1)
    segs = base + rs + ls
    spheres = []
    for off, arm in ((2, rs), (2 + len(rs), ls)):
        moving = [off + i for i, s in enumerate(arm) if s.joint_type != JOINT_FIXED]
        at = moving[:-1] + [off + len(arm) - 1]
        spheres += [_sphere(seg, (0, 0, 0), r) for seg, r in zip(at, _SPHERE_RADII)]
    return dict(n_dof=14, segments=segs, lower=rl + ll, upper=ru + lu, spheres=spheres,
                link_names=["base_link", "torso_lift_link"] + rn + ln, tool=2 + len(rs) - 1,
                tool_left=len(segs) - 1)


def spherebot():
    """trajopt_common/data/spherebot.urdf: two prismatic joints (x then y), a 0.5 m sphere."""
    segs = [_seg(-1, JOINT_PRISMATIC, 0, (0, 0, 0), (1, 0, 0)), _seg(0, JOINT_PRISMATIC, 1, (0, 0, 0), (0, 1, 0)),
            _seg(1, JOINT_FIXED, -1, (0, 0, 0))]
    return dict(n_dof=2, segments=segs, lower=[-20.0, -20.0], upper=[20.0, 20.0],
                spheres=[_sphere(2, (0, 0, 0), 0.5)], link_names=["spherebot_linkX", "spherebot_linkY", "spherebot_link"],
                tool=2)


def _copy(robot, **changes):
    out = dict(robot, segments=[Segment.from_buffer_copy(s) for s in robot["segments"]],
               spheres=[Sphere.from_buffer_copy(s) for s in robot["spheres"]], lower=list(robot["lower"]),
               upper=list(robot["upper"]), link_names=list(robot["link_names"]))
    out.update(changes)
    return out


def with_joints_fixed(robot, links):
    """`robot` with the joints of the segments named in `links` held FIXED at 0: their columns go, the later columns
    move down."""
    r = _copy(robot)
    gone = set()
    for name in links:
        s = r["segments"][r["link_names"].index(name)]
        gone.add(s.q_index)
        s.joint_type, s.q_index = JOINT_FIXED, -1
    keep = [c for c in range(robot["n_dof"]) if c not in gone]
    col = {c: i for i, c in enumerate(keep)}
    for s in r["segments"]:
        if s.q_index >= 0:
            s.q_index = col[s.q_index]
    r.update(n_dof=len(keep), lower=[r["lower"][c] for c in keep], upper=[r["upper"][c] for c in keep])
    return r


def with_joint_moving(robot, link, jtype, axis, lower, upper):
    """`robot` with the FIXED joint of segment `link` made a moving one (about / along `axis` of its frame); it takes the
    column after the robot's."""
    r = _copy(robot)
    s = r["segments"][r["link_names"].index(link)]
    assert s.joint_type == JOINT_FIXED
    s.joint_type, s.q_index = jtype, robot["n_dof"]
    s.axis[:] = axis
    r.update(n_dof=robot["n_dof"] + 1, lower=r["lower"] + [lower], upper=r["upper"] + [upper])
    return r


def on_prismatic_axes(robot, axes):
    """`robot` carried by a chain of prismatic axes [(name, axis, lower, upper)] from the scene root (the first carries
    the second, the last carries the robot's root segments).  The axes take the columns after the robot's, so their
    columns are out of segment order."""
    n, D = len(axes), robot["n_dof"]
    r = _copy(robot)
    segs = [_seg(i - 1, JOINT_PRISMATIC, D + i, (0, 0, 0), ax) for i, (_, ax, _, _) in enumerate(axes)]
    for s in r["segments"]:
        s.parent = n - 1 if s.parent < 0 else s.parent + n
    for sp in r["spheres"]:
        sp.segment += n
    r.update(n_dof=D + n, segments=segs + r["segments"], lower=r["lower"] + [a[2] for a in axes],
             upper=r["upper"] + [a[3] for a in axes], link_names=[a[0] for a in axes] + r["link_names"],
             tool=robot["tool"] + n)
    if "tool_left" in robot:
        r["tool_left"] = robot["tool_left"] + n
    return r


def linear_axis():
    """1 DOF: one prismatic axis (x, +-0.8 m) 0.5 m above the floor, carrying a 0.15 m payload sphere on a 0.2 m bracket
    and the tool frame at the payload."""
    segs = [_seg(-1, JOINT_FIXED, -1, (0, 0, 0.5)), _seg(0, JOINT_PRISMATIC, 0, (0, 0, 0), (1, 0, 0)),
            _seg(1, JOINT_FIXED, -1, (0, 0, -0.2))]
    return dict(n_dof=1, segments=segs, lower=[-0.8], upper=[0.8], spheres=[_sphere(2, (0, 0, 0), 0.15)],
                link_names=["base_link", "carriage", "payload"], tool=2)


def scara():
    """4 DOF SCARA (revolute z, revolute z, prismatic quill down, revolute z), a sphere on each link and one at the tool.
    The joint columns are out of segment order: the segments in chain order hold the columns 1, 3, 0, 2."""
    segs = [_seg(-1, JOINT_FIXED, -1, (0, 0, 0.45)),
            _seg(0, JOINT_REVOLUTE, 1, (0, 0, 0), (0, 0, 1)),
            _seg(1, JOINT_REVOLUTE, 3, (0.35, 0, 0), (0, 0, 1)),
            _seg(2, JOINT_PRISMATIC, 0, (0.3, 0, 0), (0, 0, -1)),
            _seg(3, JOINT_REVOLUTE, 2, (0, 0, -0.1), (0, 0, 1)),
            _seg(4, JOINT_FIXED, -1, (0, 0, -0.08))]
    spheres = [_sphere(1, (0.18, 0, 0), 0.08), _sphere(2, (0.15, 0, 0), 0.07), _sphere(3, (0, 0, 0), 0.05),
               _sphere(5, (0, 0, 0), 0.04)]
    return dict(n_dof=4, segments=segs, lower=[0.0, -2.5, -3.0, -2.5], upper=[0.25, 2.5, 3.0, 2.5], spheres=spheres,
                link_names=["base_link", "link1", "link2", "quill", "flange", "tool"], tool=5)


def pr2_arm_5dof():
    """The PR2 right arm with r_upper_arm_roll_joint and r_forearm_roll_joint FIXED."""
    return with_joints_fixed(pr2_arm("r"), ["r_upper_arm_roll_link", "r_forearm_roll_link"])


def pr2_arm_on_rail():
    """8 DOF: the PR2 right arm on a linear rail along x (+-0.5 m; column 7)."""
    return on_prismatic_axes(pr2_arm("r"), [("rail_x", (1, 0, 0), -0.5, 0.5)])


def pr2_arm_on_gantry():
    """9 DOF: the PR2 right arm on an x-y gantry (x carries y, +-0.5 m each; columns 7 and 8)."""
    return on_prismatic_axes(pr2_arm("r"), [("gantry_x", (1, 0, 0), -0.5, 0.5), ("gantry_y", (0, 1, 0), -0.5, 0.5)])


_DUAL_FIXED = ["r_forearm_roll_link", "l_forearm_roll_link", "l_wrist_roll_link", "r_upper_arm_roll_link"]


def pr2_dual_arm_fixed(n_fixed):
    """14 - n_fixed DOF (1 <= n_fixed <= 4): the dual arm with the first n_fixed of both forearm rolls, the left wrist roll
    and the right upper arm roll FIXED."""
    return with_joints_fixed(pr2_dual_arm(), _DUAL_FIXED[:n_fixed])


def pr2_dual_arm_on_lift(rail=False):
    """15 DOF: the dual arm with its torso lift moving (prismatic z, 0 to 0.3 m; column 14); 16 DOF with `rail`: and the
    whole robot on a linear rail along x (+-0.5 m; column 15)."""
    r = with_joint_moving(pr2_dual_arm(), "torso_lift_link", JOINT_PRISMATIC, (0, 0, 1), 0.0, 0.3)
    return on_prismatic_axes(r, [("rail_x", (1, 0, 0), -0.5, 0.5)]) if rail else r


# The robots of this module by joint count (maker functions): every count from 1 to 16 but 3 and 6
BY_JOINT_COUNT = {1: linear_axis, 2: spherebot, 4: scara, 5: pr2_arm_5dof, 7: pr2_arm,
                  8: pr2_arm_on_rail, 9: pr2_arm_on_gantry, 10: lambda: pr2_dual_arm_fixed(4),
                  11: lambda: pr2_dual_arm_fixed(3), 12: lambda: pr2_dual_arm_fixed(2),
                  13: lambda: pr2_dual_arm_fixed(1), 14: pr2_dual_arm, 15: pr2_dual_arm_on_lift,
                  16: lambda: pr2_dual_arm_on_lift(rail=True)}


SPHEREBOT_OBSTACLES = np.array([[0, 0, 0, 0.5], [-0.75, 0, 0, 0.5], [0, 0.75, 0, 0.5]], dtype=np.float64)


# ---- host-side numpy FK (problem generation only: targets = FK(q_goal), clearance checks) ----
def _quat_to_rot(q):
    w, x, y, z = np.asarray(q, float) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def fk_numpy(robot, q):
    """Frames (R[3,3], p[3]) of every segment in the scene root; mirrors tb200 FK semantics."""
    frames = []
    for s in robot["segments"]:
        R = _quat_to_rot(list(s.origin_wxyz))
        p = np.array(list(s.origin_xyz))
        if s.joint_type == JOINT_REVOLUTE:
            a = q[s.q_index]
            ax = np.array(list(s.axis))
            K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
            R = R @ (np.eye(3) + math.sin(a) * K + (1 - math.cos(a)) * (K @ K))
        elif s.joint_type == JOINT_PRISMATIC:
            p = p + R @ (np.array(list(s.axis)) * q[s.q_index])
        if s.parent >= 0:
            Rp, pp = frames[s.parent]
            R, p = Rp @ R, Rp @ p + pp
        frames.append((R, p))
    return frames


def rot_to_wxyz(R):
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        return np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
    q = np.zeros(4)
    q[1 + i] = 0.25 * s
    q[0] = (R[k, j] - R[j, k]) / s
    q[1 + j] = (R[j, i] + R[i, j]) / s
    q[1 + k] = (R[k, i] + R[i, k]) / s
    return q


def sphere_centers(robot, q):
    fr = fk_numpy(robot, q)
    return np.array([fr[s.segment][0] @ np.array(list(s.center)) + fr[s.segment][1] for s in robot["spheres"]])


def jacobian_numpy(robot, q, link):
    """6 x n_dof geometric Jacobian of segment `link`'s origin in the scene root (linear rows, then angular; a zero
    column for a joint that does not move the link): the matrix of the avoid_singularity term."""
    fr = fk_numpy(robot, q)
    segs = robot["segments"]
    J = np.zeros((6, robot["n_dof"]))
    pe = fr[link][1]
    s = link
    while s >= 0:
        g = segs[s]
        if g.joint_type != JOINT_FIXED:
            R, o = fr[s]
            a = R @ np.array(list(g.axis))
            J[:, g.q_index] = np.r_[np.cross(a, pe - o), a] if g.joint_type == JOINT_REVOLUTE else np.r_[a, 0, 0, 0]
        s = g.parent
    return J


def smallest_singular_value(robot, q, link):
    """The smallest singular value of jacobian_numpy (thin SVD: the smallest of min(6, n_dof))."""
    return float(np.linalg.svd(jacobian_numpy(robot, q, link), compute_uv=False)[-1])
