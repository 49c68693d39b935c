"""A plain high-precision reference of the convexify outputs (tb200_convexify_batch / oracle_convexify_batch).

Restated from DESIGN.md section 3 and the comments of the convexify kernel, without the oracle or the library: FK,
Jacobians, distances and pose errors are computed in np.longdouble (80-bit extended precision on x86), and every
object's value is an exactly rounded sum (math.fsum of the two-double split of each extended term).  So the reference
is more accurate than either fp64 implementation, and a mistake the kernel and the oracle share shows up against it.

`convexify(desc, x)` returns the dict of oracle_lib.convexify_batch (same row layout, same candidate order) and an
`info` dict that says which branch points the input reached (ties, clamps, filters, rotation angles), for the edge
census of tests/test_convexify_numpy.py.
"""
import math

import numpy as np

from trajopt_b200.capi import (COLL_CONTINUOUS, COLL_DISCRETE, COLL_LVS_CONTINUOUS, COLL_LVS_DISCRETE, JOINT_FIXED,
                               JOINT_PRISMATIC, JOINT_REVOLUTE, ROLE_COST, TERM_CART_POSE, TERM_CART_VEL,
                               TERM_COLLISION, TERM_JOINT_ACC, TERM_JOINT_POS, TERM_JOINT_VEL)

LD = np.longdouble
PI = LD("3.14159265358979323846264338327950288")
CART_EPS = 1e-5            # forward-difference step of the CartPose Jacobian (DEFAULT_EPSILON)
MIN_CAST_ROWS, MAX_CAST_ROWS = 128, 4096
# an error angle within PI_BAND of pi has two representatives, a0 g0 and a0 (g0 - 2 pi sign g0): which one an fp64
# implementation lands on depends on the rounding of w (info["cart_alt"] holds the other one)
PI_BAND = 1e-9


def fsum(terms):
    """The sum of extended-precision terms, correctly rounded to fp64: each term is split into hi + lo doubles."""
    parts = []
    for t in terms:
        t = LD(t)
        hi = float(t)
        parts += [hi, float(t - LD(hi))]
    return math.fsum(parts)


# ---------------------------------------------------------------------------------------------------- kinematics
def _quat_rot(wxyz):
    w, x, y, z = (LD(v) for v in wxyz)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=LD)


def fk(robot, q):
    """World frames (R, p) of every segment: origin * motion(q), composed with the parent's frame."""
    out = []
    for s in robot["segments"]:
        R = _quat_rot(list(s.origin_wxyz))
        p = np.array(list(s.origin_xyz), dtype=LD)
        ax = np.array(list(s.axis), dtype=LD)
        if s.joint_type == JOINT_REVOLUTE:
            a = LD(q[s.q_index])
            K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], dtype=LD)
            R = R @ (np.eye(3, dtype=LD) + np.sin(a) * K + (1 - np.cos(a)) * (K @ K))
        elif s.joint_type == JOINT_PRISMATIC:
            p = p + R @ (ax * LD(q[s.q_index]))
        if s.parent >= 0:
            Rp, pp = out[s.parent]
            R, p = Rp @ R, Rp @ p + pp
        out.append((R, p))
    return out


def jacobian_lin(robot, frames, link, point):
    """Translational geometric Jacobian [3][D] of a point rigidly attached to `link`: a x (point - o) for a revolute
    ancestor, a for a prismatic one, 0 for a joint that does not move the link."""
    J = np.zeros((3, robot["n_dof"]), dtype=LD)
    s = link
    while s >= 0:
        g = robot["segments"][s]
        if g.joint_type != JOINT_FIXED:
            R, o = frames[s]
            a = R @ np.array(list(g.axis), dtype=LD)
            J[:, g.q_index] = np.cross(a, point - o) if g.joint_type == JOINT_REVOLUTE else a
        s = g.parent
    return J


def sphere_centre(robot, frames, s):
    sp = robot["spheres"][s]
    R, p = frames[sp.segment]
    return R @ np.array(list(sp.center), dtype=LD) + p


def contact_normal(d, length):
    """d / |d| from the robot sphere towards the obstacle; coincident centres take (1, 0, 0) (DESIGN.md section 6)."""
    return d / length if length > 0 else np.array([1, 0, 0], dtype=LD)


# ---------------------------------------------------------------------------------------------------- pose error
def rot_decomposed(R):
    """(unit axis, signed angle in [-pi, pi]) of a rotation: the quaternion of Eigen's trace / largest-diagonal
    extraction, axis +v/|v|, the sign of w carried by the angle; the identity gives ((1, 0, 0), 0)."""
    m = R.reshape(9)
    t = m[0] + m[4] + m[8]
    q = np.zeros(4, dtype=LD)
    if t > 0:
        t = np.sqrt(t + 1)
        q[0] = t / 2
        t = LD(0.5) / t
        q[1], q[2], q[3] = (m[7] - m[5]) * t, (m[2] - m[6]) * t, (m[3] - m[1]) * t
    else:
        i = 0
        if m[4] > m[0]:
            i = 1
        if m[8] > m[i * 3 + i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1)
        q[1 + i] = t / 2
        t = LD(0.5) / t
        q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t
        q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t
        q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t
    n = np.sqrt(q[1] ** 2 + q[2] ** 2 + q[3] ** 2)
    if n == 0:
        return np.array([1, 0, 0], dtype=LD), LD(0)
    ang = 2 * np.arctan2(n, abs(q[0]))
    if q[0] < 0:
        ang = -ang
    return q[1:] / n, ang


def pose_error(target, source):
    """target^-1 * source: translation, and (axis, angle) of the rotation."""
    Rt, pt = target
    Rs, ps = source
    a, g = rot_decomposed(Rt.T @ Rs)
    return Rt.T @ (ps - pt), a, g


def fd_rot_diff(a0, g0, a1, g1):
    """Rotation part of calcJacobianTransformErrorDiff: the perturbed axis flipped to the nominal one's side (the angle
    with it), the angle moved onto the nominal one's branch by 2 pi, then a1 g1 - a0 g0."""
    flipped = a1 @ a0 < 0
    if flipped:
        a1, g1 = -a1, -g1
    diff = g1 - g0
    if diff > PI:
        g1 = g1 - 2 * PI
    elif diff < -PI:
        g1 = g1 + 2 * PI
    return a1 * g1 - a0 * g0, flipped


def _pose7(v):
    return _quat_rot(v[3:7]), np.array(v[:3], dtype=LD)


def cart_pose_rows(robot, term, target7, q, flip=False):
    """err[6] and the forward-difference Jacobian [6][D] of a CartPose term at the joint state q (unscaled, every row).
    flip: the other representative of an error rotation of angle pi (a0 g0 replaced by a0 (g0 - 2 pi sign g0)), the
    one a rounding of w to the other sign gives.  Also returns the error angle and the number of Jacobian columns whose
    perturbed axis was flipped."""
    D = robot["n_dof"]
    target = _pose7(target7)
    off = _pose7(list(term.source_offset))

    def source(qq):
        R, p = fk(robot, qq)[term.link]
        return R @ off[0], R @ off[1] + p

    e0p, a0, g0 = pose_error(target, source(q))
    if flip:
        g0 = g0 - 2 * PI * np.sign(g0)
    err = np.concatenate([e0p, a0 * g0])
    J = np.zeros((6, D), dtype=LD)
    n_flips = 0
    for j in range(D):
        qp = np.array(q, dtype=np.float64)
        qp[j] = qp[j] + CART_EPS  # (the perturbed state is the fp64 q + eps, as in both implementations)
        e1p, a1, g1 = pose_error(target, source(qp))
        J[:3, j] = (e1p - e0p) / LD(CART_EPS)
        dr, flipped = fd_rot_diff(a0, g0, a1, g1)
        J[3:, j] = dr / LD(CART_EPS)
        n_flips += flipped
    return err, J, g0, n_flips


def rotvec_error_central(robot, term, target7, q, h=1e-6):
    """An independent derivative of the rotation-vector error: scipy's Rotation, central differences in fp64."""
    from scipy.spatial.transform import Rotation
    off = _pose7(list(term.source_offset))
    Rt = np.array(_pose7(target7)[0], dtype=np.float64)

    def rv(qq):
        R = np.array(fk(robot, qq)[term.link][0] @ off[0], dtype=np.float64)
        return Rotation.from_matrix(Rt.T @ R).as_rotvec()
    D = robot["n_dof"]
    J = np.zeros((3, D))
    for j in range(D):
        e = np.zeros(D)
        e[j] = h
        J[:, j] = (rv(q + e) - rv(q - e)) / (2 * h)
    return rv(np.asarray(q, float)), J


# ---------------------------------------------------------------------------------------------------- layout
def cart_idx(term):
    """Rows a CartPose term keeps: those with |coeff| > 1e-5, positions first, with their coefficients."""
    c = list(term.pos_coeffs) + list(term.rot_coeffs)
    return [(i, c[i]) for i in range(6) if abs(c[i]) > 1e-5]


def cast_rows_per_pair(desc):
    """tb200inl_cast_rows_per_pair (include/trajopt_b200.h): every candidate of the longest initial step pair."""
    need = 1.0
    for tm in desc.terms:
        if tm.kind != TERM_COLLISION:
            continue
        if tm.evaluator_type == COLL_LVS_DISCRETE and need < 2:
            need = 2.0
        if tm.evaluator_type not in (COLL_LVS_CONTINUOUS, COLL_LVS_DISCRETE) or not tm.longest_valid_segment_length > 0:
            continue
        for b in range(desc.B):
            for t in range(max(tm.first_step, 0), tm.last_step):
                if t + 1 >= desc.T:
                    break
                s = math.sqrt(sum((desc.init_traj[b, t + 1, j] - desc.init_traj[b, t, j]) ** 2 for j in range(desc.D)))
                if s > tm.longest_valid_segment_length:
                    need = max(need, math.ceil(s / tm.longest_valid_segment_length)
                               + (1 if tm.evaluator_type == COLL_LVS_DISCRETE else 0))
    cand = math.ceil(need * len(desc.robot_spec["spheres"]) * desc.obstacles.shape[-2] / 64) * 64 \
        if desc.obstacles is not None else 0
    return int(min(max(cand, MIN_CAST_ROWS), MAX_CAST_ROWS))


def _fixed(term):
    return set(term.fixed_steps[:term.n_fixed_steps])


def _joint_eq(term, D):
    return all(abs(term.upper_tols[d]) < 1e-5 and abs(term.lower_tols[d]) < 1e-5 for d in range(D))


# ---------------------------------------------------------------------------------------------------- collision
def discrete_rows(robot, q, obs, term, info):
    """Rows {grad[D], dist0, margin, coeff | 0} of every (sphere, obstacle) candidate of one waypoint, and the hinge
    terms of the active ones in candidate order."""
    D = robot["n_dof"]
    fr = fk(robot, q)
    reach = LD(term.margin) + LD(term.margin_buffer)
    rows, vals = [], []
    for s in range(len(robot["spheres"])):
        sp = robot["spheres"][s]
        c = sphere_centre(robot, fr, s)
        J = jacobian_lin(robot, fr, sp.segment, c)
        for ob in obs:
            d = np.array(ob[:3], dtype=LD) - c
            length = np.sqrt(d @ d)
            dist = length - LD(sp.radius) - LD(ob[3])
            active = not dist > reach
            row = np.zeros(D + 3, dtype=LD)
            if active:
                row[:D] = -(contact_normal(d, length) @ J)
                vals.append(max(LD(term.margin) - dist, LD(0)) * LD(term.coeff))
            row[D], row[D + 1], row[D + 2] = dist, term.margin, term.coeff if active else 0.0
            rows.append(row)
            info["disc_tie_active"] += int(dist == reach)
            info["disc_tie_above"] += int(dist > reach and float(dist) == np.nextafter(float(reach), np.inf))
            info["coincident_discrete"] += int(length == 0 and active)
            info["disc_active"] += int(active)
    return rows, vals


def cast_rows(robot, q0, q1, obs, term, start_fixed, end_fixed, cap, info):
    """The step pair (q0, q1) of a CONTINUOUS / LVS_CONTINUOUS / LVS_DISCRETE term: its active contacts as rows
    {g0[D], g1[D], dist0, margin, coeff} in canonical order (sphere, obstacle, sub-segment), zero rows up to `cap`, and
    the hinge terms in the same order.  Returns (rows, values, n_sub, n_active); n_active > cap: the pair overflows."""
    D = robot["n_dof"]
    disc = term.evaluator_type == COLL_LVS_DISCRETE
    lvs = np.finfo(np.float64).max if term.evaluator_type == COLL_CONTINUOUS else term.longest_valid_segment_length
    q0l, q1l = np.array(q0, dtype=LD), np.array(q1, dtype=LD)
    dq = q1l - q0l
    qd = np.sqrt(dq @ dq)
    n = 1 if not qd > LD(lvs) else int(np.ceil(qd / LD(lvs)))
    info["cast_nsub"].append(n)
    info["cast_exact_multiple"] += int(n > 1 and qd == LD(n) * LD(lvs))
    info["cast_exact_lvs"] += int(qd == LD(lvs))
    info["cast_stationary"] += int(qd == 0)
    if n > 32767:
        return None, None, n, None
    states = [q0l + dq * (LD(i) / LD(n)) if i < n else q1l for i in range(n + 1)]
    frames = [fk(robot, u) for u in states]
    reach = LD(term.margin) + LD(term.margin_buffer)
    slots = n + 1 if disc else n
    cands = []
    for s, sp in enumerate(robot["spheres"]):
        for o, ob in enumerate(obs):
            c_ob = np.array(ob[:3], dtype=LD)
            for i in range(slots):
                ie = i if disc else i + 1
                ca, cb = sphere_centre(robot, frames[i], s), sphere_centre(robot, frames[ie], s)
                w = cb - ca
                ww = w @ w
                sc = (c_ob - ca) @ w / ww if ww > 0 else LD(0)
                sc = min(max(sc, LD(0)), LD(1))
                d = c_ob - (ca + sc * w)
                length = np.sqrt(d @ d)
                dist = length - LD(sp.radius) - LD(ob[3])
                time0 = i == 0 and sc == 0
                time1 = (i == n) if disc else (i == n - 1 and sc == 1)
                inside = not dist > reach
                info["time0_filtered"] += int(inside and start_fixed and time0)
                info["time1_filtered"] += int(inside and end_fixed and time1)
                info["time0_kept"] += int(inside and not start_fixed and time0 and not disc)
                info["time1_kept"] += int(inside and not end_fixed and time1 and not disc)
                info["sc_interior_clamp0"] += int(inside and i > 0 and sc == 0 and not disc)
                if not inside or (start_fixed and time0) or (end_fixed and time1):
                    continue
                info["coincident_cast"] += int(length == 0)
                cc = (LD(i) + sc) / LD(n)
                qt = q1l if cc == 1 else q0l + dq * cc
                frt = fk(robot, qt)
                Rt, pt = frt[sp.segment]
                row = np.zeros(2 * D + 3, dtype=LD)
                nrm = contact_normal(d, length)
                for k in (0, 1):
                    if (k == 0 and start_fixed) or (k == 1 and end_fixed):
                        continue
                    Rk = frames[i if disc else i + k][sp.segment][0]
                    point = Rk @ np.array(list(sp.center), dtype=LD) + pt
                    J = jacobian_lin(robot, frt, sp.segment, point)
                    row[k * D:(k + 1) * D] = -(nrm @ J) * (1 - cc if k == 0 else cc)
                row[2 * D], row[2 * D + 1], row[2 * D + 2] = dist, term.margin, term.coeff
                cands.append((row, max(LD(term.margin) - dist, LD(0)) * LD(term.coeff)))
    n_act = len(cands)
    info["cast_active"].append(n_act)
    if n_act > cap:
        return None, None, n, n_act
    rows = [r for r, _ in cands] + [np.zeros(2 * D + 3, dtype=LD)] * (cap - n_act)
    return rows, [v for _, v in cands], n, n_act


# ---------------------------------------------------------------------------------------------------- the batch
def new_info():
    return {k: 0 for k in ("disc_tie_active", "disc_tie_above", "coincident_discrete", "disc_active", "cast_exact_multiple",
                           "cast_exact_lvs", "cast_stationary", "time0_filtered", "time1_filtered", "time0_kept",
                           "time1_kept", "sc_interior_clamp0", "coincident_cast", "cart_axis_flips")} | \
        dict(cast_nsub=[], cast_active=[], cart_angle=[], overflow=[], cart_alt={})


def convexify(desc, x, bs=None):
    """The convexify outputs at x [B][T][D] for trajectories `bs` (default: all), in the layout of
    oracle_lib.convexify_batch (rows of other trajectories stay zero; collision rows of the cost objects first, then
    those of the constraints, each in term order: the objects' OptProb order).  A trajectory with a step pair beyond the row
    block (or 32767 sub-segments) is listed in info["overflow"] and its rows are left zero."""
    robot, T, D, B = desc.robot_spec, desc.T, desc.D, desc.B
    has_vel = any(t.kind == TERM_CART_VEL for t in desc.terms)
    has_cast = any(t.kind == TERM_COLLISION and t.evaluator_type != COLL_DISCRETE for t in desc.terms)
    cap = cast_rows_per_pair(desc) if has_cast else 0
    n_cart = sum(len(cart_idx(t)) if t.kind == TERM_CART_POSE else 6 * (t.last_step - t.first_step + 1)
                 for t in desc.terms if t.kind in (TERM_CART_POSE, TERM_CART_VEL))
    n_coll = 0
    for t in desc.terms:
        if t.kind == TERM_COLLISION:
            if t.evaluator_type == COLL_DISCRETE:
                n_coll += sum(1 for s in range(t.first_step, t.last_step + 1) if s not in _fixed(t)) * \
                    len(robot["spheres"]) * desc.obstacles.shape[-2]
            else:
                n_coll += (t.last_step - t.first_step) * cap
    cs, ks = (2 * D if has_vel else D), (2 * D + 3 if has_cast else D + 3)
    n_costs = n_cnts = 0
    per_term = []  # objects per term
    for t in desc.terms:
        if t.kind in (TERM_JOINT_POS, TERM_JOINT_VEL, TERM_JOINT_ACC, TERM_CART_POSE):
            k = 1
        elif t.kind == TERM_CART_VEL:
            k = t.last_step - t.first_step + 1
        elif t.kind == TERM_COLLISION and t.evaluator_type == COLL_DISCRETE:
            k = sum(1 for s in range(t.first_step, t.last_step + 1) if s not in _fixed(t))
        elif t.kind == TERM_COLLISION:
            k = t.last_step - t.first_step
        else:
            raise NotImplementedError(f"term kind {t.kind}")
        per_term.append(k)
        if t.role == ROLE_COST:
            n_costs += k
        else:
            n_cnts += k
    out = dict(cart_err=np.zeros((B, n_cart)), cart_jac=np.zeros((B, n_cart, cs)), coll_rows=np.zeros((B, n_coll, ks)),
               cost_vals=np.zeros((B, n_costs)), cnt_viols=np.zeros((B, n_cnts)))
    info = new_info()
    for b in (range(B) if bs is None else bs):
        xb = np.asarray(x[b], dtype=np.float64)
        obs = None if desc.obstacles is None else (desc.obstacles[b] if desc.c.obstacles_per_traj else
                                                   desc.obstacles.reshape(-1, desc.obstacles.shape[-2], 4)[0])
        cart_r = coll_r = ic = ik = 0
        costs, cnts = [], []
        blocks = ([], [])  # collision rows of the cost objects, of the constraints: written in that order
        overflow = False
        for term, n_obj in zip(desc.terms, per_term):
            is_cost = term.role == ROLE_COST
            vals = []  # one value per object
            if term.kind in (TERM_JOINT_POS, TERM_JOINT_VEL, TERM_JOINT_ACC):
                order = term.kind - TERM_JOINT_POS
                w = [[1], [-1, 1], [1, -2, 1]][order]
                es = [(sum(LD(w[k]) * LD(xb[i + k, j]) for k in range(order + 1)) - LD(term.targets[j]), j)
                      for i in range(term.first_step, term.last_step + 1 - order) for j in range(D)]
                if _joint_eq(term, D):  # value e^2 c, also for the constraint (whose rows are c e): the quirk kept
                    terms = [e * e * LD(term.coeffs[j]) for e, j in es]
                    vals.append(fsum(terms) if is_cost else fsum(abs(v) for v in terms))
                else:
                    terms = []
                    for e, j in es:
                        terms += [max((e - LD(term.upper_tols[j])) * LD(term.coeffs[j]), LD(0)),
                                  max((LD(term.lower_tols[j]) - e) * LD(term.coeffs[j]), LD(0))]
                    vals.append(fsum(terms))
            elif term.kind == TERM_CART_POSE:
                tgt = desc.cart_targets[b, term.target_slot] if term.target_slot >= 0 else list(term.target_pose)
                t = term.first_step
                err, J, g0, n_flips = cart_pose_rows(robot, term, tgt, xb[t])
                info["cart_angle"].append(float(g0))
                info["cart_axis_flips"] += n_flips
                if abs(g0) > PI - LD(PI_BAND):  # the other representative at pi, scaled rows as below
                    ea, Ja, _, _ = cart_pose_rows(robot, term, tgt, xb[t], flip=True)
                    info["cart_alt"][(b, cart_r)] = (np.array([ea[i] * LD(c) for i, c in cart_idx(term)], np.float64),
                                                     np.array([Ja[i] * LD(c) for i, c in cart_idx(term)], np.float64))
                terms = []
                for i, c in cart_idx(term):
                    out["cart_err"][b, cart_r] = err[i] * LD(c)
                    out["cart_jac"][b, cart_r, :D] = J[i] * LD(c)
                    # EQ violation |c e|; the ABS cost c |e| (the coefficient after the abs: negative for c < 0)
                    terms.append(LD(c) * abs(err[i]) if is_cost else abs(err[i] * LD(c)))
                    cart_r += 1
                vals.append(fsum(terms))
            elif term.kind == TERM_CART_VEL:
                for t in range(term.first_step, term.last_step + 1):
                    f0, f1 = fk(robot, xb[t]), fk(robot, xb[t + 1])
                    p0, p1 = f0[term.link][1], f1[term.link][1]
                    J0, J1 = jacobian_lin(robot, f0, term.link, p0), jacobian_lin(robot, f1, term.link, p1)
                    lim = LD(term.max_displacement)
                    err = np.concatenate([p1 - p0 - lim, p0 - p1 - lim])
                    out["cart_err"][b, cart_r:cart_r + 6] = err
                    out["cart_jac"][b, cart_r:cart_r + 3, :D] = -J0
                    out["cart_jac"][b, cart_r:cart_r + 3, D:2 * D] = J1
                    out["cart_jac"][b, cart_r + 3:cart_r + 6, :D] = J0
                    out["cart_jac"][b, cart_r + 3:cart_r + 6, D:2 * D] = -J1
                    cart_r += 6
                    vals.append(fsum(abs(e) for e in err) if is_cost else fsum(max(e, LD(0)) for e in err))
            elif term.evaluator_type == COLL_DISCRETE:
                for t in range(term.first_step, term.last_step + 1):
                    if t in _fixed(term):
                        continue
                    rows, v = discrete_rows(robot, xb[t], obs, term, info)
                    blocks[not is_cost].append(np.array(rows, dtype=np.float64).reshape(-1, ks))
                    coll_r += len(rows)
                    vals.append(fsum(v))
            else:
                for t in range(term.first_step, term.last_step):
                    sf = t in _fixed(term)
                    ef = not sf and (t + 1) in _fixed(term)
                    rows, v, _, _ = cast_rows(robot, xb[t], xb[t + 1], obs, term, sf, ef, cap, info)
                    if rows is None:
                        overflow = True
                        rows, v = [], []
                    blocks[not is_cost].append(np.array(rows, dtype=np.float64).reshape(-1, ks) if rows else
                                               np.zeros((cap, ks)))
                    coll_r += cap
                    vals.append(fsum(v))
            assert len(vals) == n_obj
            if is_cost:
                costs.extend(vals)
            else:  # OptProb lists the EQ constraints (joint Eq, CartPose) before the INEQ ones, each in term order
                eq = term.kind == TERM_CART_POSE or (term.kind in (TERM_JOINT_POS, TERM_JOINT_VEL, TERM_JOINT_ACC)
                                                     and _joint_eq(term, D))
                cnts.extend((not eq, len(cnts), v) for v in vals)
        if blocks[0] or blocks[1]:
            out["coll_rows"][b] = np.concatenate(blocks[0] + blocks[1])
        if overflow:
            info["overflow"].append(b)
            out["coll_rows"][b] = 0
        out["cost_vals"][b] = costs
        out["cnt_viols"][b] = [v for _, _, v in sorted(cnts, key=lambda c: c[:2])]
        ic, ik = len(costs), len(cnts)
        assert (ic, ik, cart_r, coll_r) == (n_costs, n_cnts, n_cart, n_coll)
    return out, info
