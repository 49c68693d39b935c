"""The trajectory collision check (tb200_check_trajectories; Problem.check, api.check; checkTrajectories in C++): what
tesseract's checkTrajectory answers for the reference's collision tests, for every trajectory of a batch.

CPU: a CPU model of the check (tests/cpp/check_oracle.cpp, built on the oracle's robot model) equals a plain-numpy
restatement of the four types (per-slot minimum, contacts, argmin and the per-trajectory summary), the LVS types bound
each other as they must, and the reference's before / after expectations hold on the repo's copies of its problem files
solved by the oracle.  GPU: the device equals the CPU model on the same cases and on a configs[2] batch of 1024, x = None
checks the last solve's x, the reference files solved on the device pass the same expectations, refusals come with
their messages, and the C++ layer returns the C ABI's values."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import cpp_host
from trajopt_b200 import capi, problems, robots
from test_reference_json import _load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = [capi.COLL_DISCRETE, capi.COLL_LVS_DISCRETE, capi.COLL_CONTINUOUS, capi.COLL_LVS_CONTINUOUS]


# ---- CPU model of the check (tests/cpp/check_oracle.cpp over the oracle's robot model) -------------------------------
class CheckOracle:
    def __init__(self, path):
        self.lib = C.CDLL(path)

    def check_trajectories(self, desc, x, type, lvs=0.005, margin=0.0):
        """The check of x [B][T][D] on the CPU; the same dict as api.Problem.check."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        S = desc.T if type == capi.COLL_DISCRETE else max(desc.T - 1, 0)
        out = dict(step_min_distance=np.zeros((desc.B, S)), step_contacts=np.zeros((desc.B, S), np.int32),
                   step_argmin=np.zeros((desc.B, S, 3), np.int32), in_collision=np.zeros(desc.B, np.int32),
                   first_slot=np.zeros(desc.B, np.int32), min_distance=np.zeros(desc.B))
        ptr = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32) if a.dtype == np.int32 else C.POINTER(C.c_double))  # noqa: E731
        rc = self.lib.check_oracle_trajectories(C.byref(desc.c), 0, desc.B, ptr(x), C.c_int(type), C.c_double(lvs),
                                                C.c_double(margin), *[ptr(v) for v in out.values()])
        assert rc == 0
        out["in_collision"] = out["in_collision"].astype(bool)
        return out


@pytest.fixture(scope="module")
def chk(oracle, tmp_path_factory):
    lib = os.path.join(ROOT, "oracle", "liboracle.so")
    # the oracle's own flags (oracle/Makefile)
    flags = ("-O3", "-march=x86-64-v3", "-fopenmp", "-DNDEBUG", "-I", os.path.join(ROOT, "oracle"), lib,
             "-Wl,-rpath," + os.path.dirname(lib))
    return CheckOracle(cpp_host.build(tmp_path_factory, "check_oracle", shared=True, extra=flags))


# ---- plain-numpy restatement -------------------------------------------------------------------------------------
def _sub_segments(q0, q1, lvs):
    d2 = 0.0
    for a, b in zip(q0, q1):  # (sequential, as the C++ and CUDA code add them)
        d2 += (b - a) * (b - a)
    qd = math.sqrt(d2)
    return int(math.ceil(qd / lvs)) if math.isfinite(qd) and qd > lvs else 1


def _swept(pa, pb, r, ob):
    """[L][O] distances of the spheres moving on the chords pa -> pb ([L][3]) to the obstacles ob ([O][4])."""
    w = pb - pa
    ww = np.einsum("lk,lk->l", w, w)[:, None]
    wd = np.einsum("lok,lk->lo", ob[None, :, :3] - pa[:, None, :], w)
    s = np.clip(np.divide(wd, ww, out=np.zeros_like(wd), where=ww > 0), 0.0, 1.0)[:, :, None]
    p = np.where(s == 1.0, pb[:, None, :], pa[:, None, :] + s * w[:, None, :])
    return np.linalg.norm(ob[None, :, :3] - p, axis=2) - r[:, None] - ob[None, :, 3]


def numpy_check(desc, x, type, lvs=0.005, margin=0.0):
    rob = desc.robot_spec
    r = np.array([s.radius for s in rob.get("spheres", [])])
    T, B = desc.T, desc.B
    S = T if type == capi.COLL_DISCRETE else T - 1
    swept = type in (capi.COLL_CONTINUOUS, capi.COLL_LVS_CONTINUOUS)
    out = dict(step_min_distance=np.zeros((B, S)), step_contacts=np.zeros((B, S), np.int32),
               step_argmin=np.full((B, S, 3), -1, np.int32))
    for b in range(B):
        ob = np.zeros((0, 4)) if desc.obstacles is None else (desc.obstacles[b] if desc.c.obstacles_per_traj else desc.obstacles)
        for t in range(S):
            q0 = x[b, t]
            q1 = q0 if type == capi.COLL_DISCRETE else x[b, t + 1]
            n = _sub_segments(q0, q1, lvs) if type in (capi.COLL_LVS_DISCRETE, capi.COLL_LVS_CONTINUOUS) else 1
            n_tests = 1 if type == capi.COLL_DISCRETE else (n if swept else n + 1)
            if len(r) == 0 or len(ob) == 0:
                out["step_min_distance"][b, t] = np.inf
                continue
            states = [q0 if i == 0 else (q1 if i == n else q0 + (q1 - q0) * (i / n)) for i in range(n_tests + swept)]
            cen = [robots.sphere_centers(rob, q) for q in states]
            d = np.stack([_swept(cen[i], cen[i + 1] if swept else cen[i], r, ob) for i in range(n_tests)], axis=2)
            fin = np.isfinite(d)
            v = np.where(fin, d, -np.inf).ravel()  # (sphere, obstacle, sub) order; argmin takes the first minimum
            k = int(np.argmin(v))
            out["step_min_distance"][b, t] = np.nan if v[k] == -np.inf else v[k]
            out["step_contacts"][b, t] = int((~(fin & (d >= margin))).sum())
            out["step_argmin"][b, t] = np.unravel_index(k, d.shape)
    c = out["step_contacts"]
    out["in_collision"] = (c > 0).any(axis=1)
    out["first_slot"] = np.where(out["in_collision"], np.argmax(c > 0, axis=1), -1).astype(np.int32)
    m = out["step_min_distance"]
    out["min_distance"] = np.where(np.isnan(m).any(axis=1), np.nan, np.min(np.where(np.isnan(m), np.inf, m), axis=1, initial=np.inf))
    return out


def candidate_distance(desc, x, type, lvs, b, t, key):
    """Distance of one candidate (sphere, obstacle, sub-index) of slot t of trajectory b, by the numpy restatement."""
    s, o, i = (int(v) for v in key)
    q0 = x[b, t]
    q1 = q0 if type == capi.COLL_DISCRETE else x[b, t + 1]
    n = _sub_segments(q0, q1, lvs) if type in (capi.COLL_LVS_DISCRETE, capi.COLL_LVS_CONTINUOUS) else 1
    state = lambda k: q0 if k == 0 else (q1 if k == n else q0 + (q1 - q0) * (k / n))  # noqa: E731
    rob = desc.robot_spec
    ob = (desc.obstacles[b] if desc.c.obstacles_per_traj else desc.obstacles)[o:o + 1]
    r = np.array([rob["spheres"][s].radius])
    ca = robots.sphere_centers(rob, state(i))[s:s + 1]
    cb = robots.sphere_centers(rob, state(i + 1))[s:s + 1] if type in (capi.COLL_CONTINUOUS, capi.COLL_LVS_CONTINUOUS) else ca
    return float(_swept(ca, cb, r, ob)[0, 0])


def assert_same(got, want, atol=1e-12, tie=None):
    """Equal results.  With tie = (desc, x, type, lvs): where the argmins differ, the two candidates must be tied to within
    atol (solved trajectories hold active constraints at the same distance, and two FKs that round differently may
    order such candidates either way)."""
    for k in ("step_contacts", "in_collision", "first_slot"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    diff = np.argwhere((got["step_argmin"] != want["step_argmin"]).any(axis=2))
    if tie is None or len(diff) > 8:
        np.testing.assert_array_equal(got["step_argmin"], want["step_argmin"], err_msg="step_argmin")
    for b, t in diff:
        a, w = (candidate_distance(*tie, b, t, r["step_argmin"][b, t]) for r in (got, want))
        assert abs(a - w) <= atol, (b, t, got["step_argmin"][b, t], want["step_argmin"][b, t], a, w)
    for k in ("step_min_distance", "min_distance"):
        np.testing.assert_allclose(got[k], want[k], rtol=0, atol=atol, equal_nan=True, err_msg=k)


# ---- cases -----------------------------------------------------------------------------------------------------------
def _perturbed(desc, seed, scale=0.15):
    """The initial trajectories with a random wiggle of the interior waypoints (more contacts, uneven step lengths)."""
    x = desc.init_traj.copy()
    x[:, 1:-1] += np.random.default_rng(seed).normal(0.0, scale, x[:, 1:-1].shape)
    return x


def _spherebot_long():
    """spherebot through the three obstacles of simple_collision_test in two long steps: > 200 sub-segments a pair."""
    rob = robots.spherebot()
    x = np.array([[[-1.9, 0.0], [0.4, 0.1], [1.9, 3.8]], [[-0.75, 0.75], [-0.75, 0.75], [0.0, -2.0]]])
    d = capi.ProblemDesc(rob, 3, [], x, obstacles=np.repeat(robots.SPHEREBOT_OBSTACLES[None], 2, axis=0))
    return d, x


CASES = {  # name -> (description, x, lvs, margin)
    "cfg2": lambda: (lambda d: (d, _perturbed(d, 1), 0.05, 0.02))(problems.config2(B=4, T=30)),
    "cfg3": lambda: (lambda d: (d, _perturbed(d, 2), 0.05, 0.0))(problems.config3(B=3, T=20)),
    "variants": lambda: (lambda d: (d, _perturbed(d, 3), 0.1, 0.05))(problems.config_variants(B=3, T=10)),
    "spherebot": lambda: (lambda d: (d[0], d[1], 0.01, 0.0))(_spherebot_long()),
    "cfg4": lambda: (lambda d: (d, _perturbed(d, 4), 0.1, 0.1))(problems.config4(B=3, T=12)),
}
_cache = {}


def case(name):
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]


# ---- CPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("type", TYPES)
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_numpy(chk, name, type):
    d, x, lvs, margin = case(name)
    got = chk.check_trajectories(d, x, type, lvs, margin)
    assert_same(got, numpy_check(d, x, type, lvs, margin))
    if type == capi.COLL_DISCRETE:
        assert got["in_collision"].any()  # (the cases do touch the obstacles)


def test_cases_reach_long_pairs():
    d, x, lvs, _ = case("spherebot")
    assert max(_sub_segments(x[b, t], x[b, t + 1], lvs) for b in range(d.B) for t in range(d.T - 1)) > 200


def test_non_finite_and_empty(chk):
    """A non-finite distance is a contact and reads NaN; a world without obstacles gives +inf and no contacts."""
    d, x, lvs, _ = case("cfg2")
    y = x.copy()
    y[1, 5, 2] = np.nan
    y[2, 7, 0] = np.inf
    for type in TYPES:
        got, fin = chk.check_trajectories(d, y, type, lvs), chk.check_trajectories(d, x, type, lvs)
        for k in got:  # the other trajectories are untouched
            np.testing.assert_array_equal(got[k][[0, 3]], fin[k][[0, 3]], err_msg=k)
        assert np.isnan(got["min_distance"][1:3]).all() and got["in_collision"][1:3].all()
        bad = [5] if type == capi.COLL_DISCRETE else [4, 5]  # the slots that read waypoint 5 of trajectory 1
        assert np.isnan(got["step_min_distance"][1, bad]).all() and (got["step_contacts"][1, bad] > 0).all()
    empty = capi.ProblemDesc(d.robot_spec, d.T, [], x)  # no obstacles
    got = chk.check_trajectories(empty, x, capi.COLL_LVS_CONTINUOUS, lvs)
    assert np.isinf(got["step_min_distance"]).all() and (got["step_contacts"] == 0).all()
    assert (got["step_argmin"] == -1).all() and (got["first_slot"] == -1).all() and not got["in_collision"].any()


@pytest.mark.parametrize("name", list(CASES))
def test_lvs_types_bound_each_other(chk, name):
    """A swept sub-segment is never farther than the states at its ends; DISCRETE is the sub-states 0 and n."""
    d, x, lvs, margin = case(name)
    disc = chk.check_trajectories(d, x, capi.COLL_DISCRETE, lvs, margin)
    ld = chk.check_trajectories(d, x, capi.COLL_LVS_DISCRETE, lvs, margin)
    lc = chk.check_trajectories(d, x, capi.COLL_LVS_CONTINUOUS, lvs, margin)
    assert (ld["step_min_distance"] >= lc["step_min_distance"] - 1e-12).all()
    assert (ld["step_min_distance"] <= np.minimum(disc["step_min_distance"][:, :-1], disc["step_min_distance"][:, 1:])).all()
    # one sub-segment per pair: LVS_DISCRETE tests exactly the two waypoints
    big = chk.check_trajectories(d, x, capi.COLL_LVS_DISCRETE, 1e9, margin)
    dm = disc["step_min_distance"]
    np.testing.assert_array_equal(big["step_min_distance"], np.minimum(dm[:, :-1], dm[:, 1:]))
    np.testing.assert_array_equal(big["step_contacts"], disc["step_contacts"][:, :-1] + disc["step_contacts"][:, 1:])
    second = dm[:, 1:] < dm[:, :-1]
    np.testing.assert_array_equal(big["step_argmin"][:, :, 2], second.astype(np.int32))
    np.testing.assert_array_equal(big["step_argmin"][:, :, :2], np.where(second[..., None], disc["step_argmin"][:, 1:, :2],
                                                                        disc["step_argmin"][:, :-1, :2]))


def _reference_check(name):
    """The type, lvs and margin the reference's test of this file checks with."""
    if name == "simple_collision_test":
        return capi.COLL_DISCRETE, 0.005, 0.2
    d = _load(name)
    coll = [t for t in d.terms if t.kind == capi.TERM_COLLISION][0]
    assert coll.evaluator_type in (capi.COLL_CONTINUOUS, capi.COLL_LVS_CONTINUOUS)
    return coll.evaluator_type, coll.longest_valid_segment_length, 0.0


REF_FILES = ["simple_collision_test", "box_cast_test", "arm_around_table"]


def assert_reference_expectation(name, check, x0, x1):
    """Contacts before the solve, none after.  arm_around_table: the obstacle sphere that stands in for the table overlaps
    the goal state itself, which the file fixes (fixed_steps [0, 5]) and no solve can move.  There the initial
    trajectory is in contact before its last step pair, and after the solve the only contact is the goal: contacts in the
    last pair alone, at the DISCRETE distance of the goal waypoint."""
    type, lvs, margin = _reference_check(name)
    before, after = check(x0, type, lvs, margin), check(x1, type, lvs, margin)
    if name != "arm_around_table":
        assert before["in_collision"].all()
        assert not after["in_collision"].any(), after["min_distance"]
        return
    goal = check(x1, capi.COLL_DISCRETE, lvs, margin)["step_min_distance"][0, -1]
    assert goal < 0
    assert (before["step_contacts"][0, :-1] > 0).any()
    assert (after["step_contacts"][0, :-1] == 0).all() and after["step_contacts"][0, -1] > 0
    np.testing.assert_allclose(after["step_min_distance"][0, -1], goal, rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", REF_FILES)
def test_reference_expectations_on_the_oracle(oracle, chk, name):
    d = _load(name)
    r = oracle.solve_batch(d)
    assert (r["status"] == capi.OPT_CONVERGED).all()
    assert_reference_expectation(name, lambda x, *a: chk.check_trajectories(d, x, *a), d.init_traj, r["x"])


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_matches_oracle(chk, name):
    from trajopt_b200 import api
    d, x, lvs, margin = case(name)
    p = api.Problem(d)
    try:
        for type in TYPES:
            assert_same(p.check(x, type=type, lvs=lvs, margin=margin), chk.check_trajectories(d, x, type, lvs, margin))
        y = x.copy()
        y[0, 1, 0] = np.nan
        y[-1, 2, 1] = -np.inf
        for type in TYPES:
            assert_same(p.check(y, type=type, lvs=lvs, margin=margin), chk.check_trajectories(d, y, type, lvs, margin))
    finally:
        p.close()


@pytest.mark.gpu
def test_device_without_obstacles(chk):
    from trajopt_b200 import api
    d, x, lvs, _ = case("cfg2")
    empty = capi.ProblemDesc(d.robot_spec, d.T, [], x)
    for type in TYPES:
        got = api.check(empty, x, type=type, lvs=lvs)
        assert_same(got, chk.check_trajectories(empty, x, type, lvs))
        assert np.isinf(got["min_distance"]).all() and not got["in_collision"].any()


@pytest.fixture(scope="module")
def cfg2_solved():
    from trajopt_b200 import api
    d = problems.config2(B=1024, T=30)
    p = api.Problem(d)
    p.solve_resident()
    yield d, p, p.fetch()
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("type", TYPES)
def test_device_matches_oracle_on_a_cfg2_batch(chk, cfg2_solved, type):
    d, p, res = cfg2_solved
    for x in (d.init_traj, res["x"]):
        assert_same(p.check(x, type=type, lvs=0.01), chk.check_trajectories(d, x, type, 0.01), tie=(d, x, type, 0.01))


@pytest.mark.gpu
@pytest.mark.parametrize("type", TYPES)
def test_none_checks_the_last_solve(cfg2_solved, type):
    d, p, res = cfg2_solved
    resident = p.check(None, type=type, lvs=0.01)
    passed = p.check(res["x"], type=type, lvs=0.01)
    for k in passed:
        np.testing.assert_array_equal(resident[k], passed[k], err_msg=k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", REF_FILES)
def test_reference_expectations_on_the_device(name):
    from trajopt_b200 import api
    d = _load(name)
    p = api.Problem(d)
    try:
        r = p.solve()
        assert (r["status"] == capi.OPT_CONVERGED).all()
        check = lambda x, type, lvs, margin: p.check(x, type=type, lvs=lvs, margin=margin)  # noqa: E731
        assert_reference_expectation(name, check, d.init_traj, None)  # x = None: the solve's x on the device
    finally:
        p.close()


@pytest.mark.gpu
def test_refusals():
    from trajopt_b200 import api
    d, x, _, _ = case("variants")
    p = api.Problem(d)
    try:
        for kw, msg in [(dict(x=None), "no solve"), (dict(x=x, type=0), "unknown collision check type"),
                        (dict(x=x, type=5), "unknown collision check type"),
                        (dict(x=x, type=capi.COLL_LVS_DISCRETE, lvs=0.0), "longest_valid_segment_length"),
                        (dict(x=x, type=capi.COLL_LVS_CONTINUOUS, lvs=-1.0), "longest_valid_segment_length"),
                        (dict(x=x, type=capi.COLL_LVS_CONTINUOUS, lvs=float("nan")), "longest_valid_segment_length"),
                        (dict(x=x, margin=float("inf")), "margin")]:
            with pytest.raises(RuntimeError) as e:
                p.check(**kw)
            assert f"error {capi.ERR_INVALID}:" in str(e.value) and msg in str(e.value), (kw, str(e.value))
        # the non-LVS types ignore lvs
        p.check(x, type=capi.COLL_CONTINUOUS, lvs=0.0)
    finally:
        p.close()


# ---- C++ host layer ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "check_host")


def test_host_program_builds(host_bin):
    assert os.access(host_bin, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("type", TYPES)
def test_cpp_layer_returns_the_c_abi_values(host_bin, tmp_path, type):
    from trajopt_b200 import api
    d, x, lvs, margin = case("cfg2")
    # (the same description without terms: which fixed segments the host folds, and so the FK's products, match)
    e = capi.ProblemDesc(d.robot_spec, d.T, [], x, obstacles=d.obstacles)
    out = subprocess.run([host_bin, cpp_host.write_problem(tmp_path / "in.txt", e), str(type), repr(lvs), repr(margin)],
                         capture_output=True, text=True, check=True).stdout.split("\n")
    want = api.check(e, x, type=type, lvs=lvs, margin=margin)
    for b in range(d.B):
        v = out[b].split()
        assert int(v[0]) == int(want["in_collision"][b]) and int(v[1]) == want["first_slot"][b]
        assert float(v[2]) == want["min_distance"][b]
        S = want["step_contacts"].shape[1]
        assert [float(t) for t in v[3:3 + S]] == want["step_min_distance"][b].tolist()
        assert [int(t) for t in v[3 + S:3 + 2 * S]] == want["step_contacts"][b].tolist()
