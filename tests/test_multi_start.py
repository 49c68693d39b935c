"""Multi-start solves (tb200_problem_desc.group_size / group_stop; DESIGN.md sections 4.1 and 6).

A group is G contiguous trajectories, the seeds of one problem.  With group_stop a seed that ends OPT_CONVERGED by its
own SQP ends its running siblings at their next SQP iteration top, under the time-limit rule; the best seed of every
group is selected on the device by the key (status != OPT_CONVERGED, max(cnt_viols) when not converged, total_cost,
index), NaN read as +inf.  `select_cpu` below restates that key; the CPU model of an early-ended run is the oracle's
SQP driver with its QP-budget stop rule (oracle_lib.solve_batch(..., qp_budget=)).
CPU: validation before the device, the key on synthetic results, seed_trajectories, sharding on group boundaries, the
C++ layer's flattening.  GPU (-m gpu): the device against the ungrouped solve, the CPU selection and the CPU model."""
import ctypes as C
import os
import socket
import subprocess

import numpy as np
import pytest

from trajopt_b200 import api, capi, problems, sharding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "trajopt_b200", "csrc")
_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)
RESULT_KEYS = ("status", "n_qp_solves", "n_func_evals", "n_admm_iters", "x", "total_cost", "cost_vals", "cnt_viols")


# ---------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    capi.load_library()  # the CUDA build must exist (no GPU needed to load it)
    out = str(tmp_path_factory.mktemp("mscpp") / "multi_start_host")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "multi_start_host.cpp"), "-o", out, "-L", CSRC, "-ltrajopt_b200",
           "-Wl,-rpath," + CSRC, "-Wl,--allow-shlib-undefined"]
    subprocess.run(cmd, check=True)
    return out


def seeded(make, n_seeds, group_stop=0, seed=7, spread=0.6):
    return problems.with_seeds(make(), n_seeds, np.random.default_rng(seed), spread, group_stop=group_stop)


def cfg2_seeded(n_seeds=8, group_stop=0):
    return seeded(lambda: problems.config2(B=32, T=30), n_seeds, group_stop)


def cfg3_seeded(n_seeds=4, group_stop=0):
    return seeded(lambda: problems.config3(B=8, T=30), n_seeds, group_stop)


def select_cpu(status, cnt_viols, total_cost, G):
    """The selection key restated: per group the argmin of (not converged, max violation when not converged, total
    cost, index) with NaN as +inf; also the number of converged seeds."""
    B = len(status)
    G = max(G, 1)
    inf = lambda v: np.where(np.isnan(v), np.inf, v)  # noqa: E731
    viol = np.zeros(B) if cnt_viols.shape[1] == 0 else inf(cnt_viols).max(axis=1)
    failed = status != capi.OPT_CONVERGED
    keys = [(int(failed[b]), float(viol[b]) if failed[b] else 0.0, float(inf(total_cost[b])), b) for b in range(B)]
    best = np.array([min(keys[g * G:(g + 1) * G])[3] for g in range(B // G)], np.int32)
    n_conv = (~failed).reshape(-1, G).sum(axis=1).astype(np.int32)
    return best, n_conv


# --------------------------------------------------------------------------------------------------------------- CPU
def _create(d):
    lib = capi.load_library()
    h = C.c_void_p()
    rc = lib.tb200_problem_create(C.byref(d.c), 0, C.byref(h))
    if rc == 0:
        lib.tb200_problem_destroy(h)
    return rc, lib.tb200_last_error().decode()


@pytest.mark.parametrize("G,stop,msg", [(-1, 0, "group_size must be >= 0"), (3, 0, "not a multiple of group_size"),
                                        (16, 1, "not a multiple of group_size"), (2, 2, "group_stop must be 0 or 1"),
                                        (4, -1, "group_stop must be 0 or 1")])
def test_bad_group_settings_are_refused_before_the_device(G, stop, msg):
    d = problems.config2(B=8, T=10)
    d.c.group_size, d.c.group_stop = G, stop
    rc, err = _create(d)
    assert rc == capi.ERR_INVALID and msg in err


@pytest.mark.parametrize("G,stop", [(0, 0), (0, 1), (1, 1), (2, 1), (4, 0), (8, 1)])
def test_good_group_settings_reach_the_device(G, stop):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    d = problems.config2(B=8, T=10)
    d.c.group_size, d.c.group_stop = G, stop
    rc, err = _create(d)
    assert rc == capi.ERR_NO_DEVICE and "no CPU fallback" in err


def test_selection_key_on_synthetic_results():
    C_, S, P = capi.OPT_CONVERGED, capi.OPT_SCO_ITERATION_LIMIT, capi.OPT_PENALTY_ITERATION_LIMIT
    nan, inf = float("nan"), float("inf")
    status = np.array([S, C_, C_, P,     # 0: two converged seeds with equal cost: the lower index
                       P, S, P, S,       # 1: none converged: the smallest worst violation, then the cost
                       C_, C_, S, C_,    # 2: a NaN cost loses to any finite cost; a failed seed never beats a converged one
                       S, P, S, S])      # 3: NaN violations read as +inf; ties on violation go to cost, then index
    viols = np.array([[0, 0], [9, 9], [9, 9], [0, 0],
                      [0.3, 0.1], [0.2, 0.2], [0.1, 0.2], [0.2, 0.05],
                      [0, 0], [0, 0], [0, 0], [0, 0],
                      [nan, 0], [0.5, 0.5], [0.5, 0.1], [0.5, 0.2]])
    cost = np.array([0.1, 2.0, 2.0, 0.0,
                     1.0, 5.0, 3.0, 4.0,
                     nan, 7.0, -1.0, 6.0,
                     0.0, 2.0, 1.0, 1.0])
    best, n_conv = select_cpu(status, viols, cost, 4)
    np.testing.assert_array_equal(best, [1, 6, 11, 14])
    np.testing.assert_array_equal(n_conv, [2, 0, 3, 0])
    # G = B: one group; G = 1 (and 0): every trajectory is its own group
    assert select_cpu(status, viols, cost, 16)[0].tolist() == [1]
    assert select_cpu(status, viols, cost, 16)[1].tolist() == [5]
    for G in (0, 1):
        best, n_conv = select_cpu(status, viols, cost, G)
        np.testing.assert_array_equal(best, np.arange(16))
        np.testing.assert_array_equal(n_conv, (status == C_).astype(np.int32))
    # all costs NaN and no converged seed: the violation decides, then the index
    assert select_cpu(np.full(3, S), np.array([[1.0], [0.5], [0.5]]), np.full(3, nan), 3)[0].tolist() == [1]
    assert select_cpu(np.full(2, S), np.array([[inf], [nan]]), np.zeros(2), 2)[0].tolist() == [0]


def test_seed_trajectories():
    d = problems.config2(B=5, T=12)
    lo, hi = np.array(d.robot_spec["lower"]), np.array(d.robot_spec["upper"])
    start, goal = d.init_traj[:, 0], d.init_traj[:, -1]
    a = problems.seed_trajectories(start, goal, 12, 6, np.random.default_rng(3), 2.0, lo, hi)
    b = problems.seed_trajectories(start, goal, 12, 6, np.random.default_rng(3), 2.0, lo, hi)
    c = problems.seed_trajectories(start, goal, 12, 6, np.random.default_rng(4), 2.0, lo, hi)
    assert a.shape == (30, 12, 7)
    np.testing.assert_array_equal(a, b)  # deterministic per rng
    assert not np.array_equal(a, c)
    g = a.reshape(5, 6, 12, 7)
    np.testing.assert_array_equal(g[:, 0], problems.interpolate(start, goal, 12))  # seed 0: the straight line
    np.testing.assert_array_equal(g[:, :, 0], np.repeat(start[:, None], 6, axis=1))  # endpoints kept exactly
    np.testing.assert_array_equal(g[:, :, -1], np.repeat(goal[:, None], 6, axis=1))
    assert (a >= lo).all() and (a <= hi).all()  # a spread of 2 rad reaches the limits: clamped
    mid = g[:, 1:, (12 - 1) // 2]
    assert (np.abs(mid - 0.5 * (start + goal)[:, None]) <= 2.0 + 1e-12).all()
    assert len({tuple(np.round(m, 12).ravel()) for m in g[0]}) == 6  # the seeds differ
    # one problem as a flat vector works too, and a single seed is the straight line
    one = problems.seed_trajectories(start[0], goal[0], 12, 1, np.random.default_rng(0), 0.5)
    np.testing.assert_array_equal(one[0], problems.interpolate(start[:1], goal[:1], 12)[0])


def test_with_seeds_repeats_the_problem_data():
    base = problems.config2(B=3, T=10)
    d = seeded(lambda: base, 4, group_stop=1)
    assert (d.B, d.c.group_size, d.c.group_stop) == (12, 4, 1)
    np.testing.assert_array_equal(d.obstacles, np.repeat(base.obstacles, 4, axis=0))
    np.testing.assert_array_equal(d.cart_targets, np.repeat(base.cart_targets, 4, axis=0))
    assert bytes(d._terms) == bytes(base._terms)
    with pytest.raises(ValueError, match="splits a group"):
        d.slice(2, 8)
    s = d.slice(4, 12)
    assert (s.B, s.c.group_size, s.c.group_stop) == (8, 4, 1)


def test_shard_bounds_keep_groups_whole():
    for groups in (1, 3, 5, 8):
        for G in (2, 4, 8):
            for world in (1, 2, 3, 4):
                spans = [sharding.shard_bounds(groups * G, r, world, G) for r in range(world)]
                assert spans[0][0] == 0 and spans[-1][1] == groups * G
                assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
                assert all(b0 % G == 0 and b1 % G == 0 for b0, b1 in spans)
                sizes = [(b - a) // G for a, b in spans]
                assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        sharding.shard_bounds(10, 0, 2, 4)
    assert sharding.converged_count([0, 1, 1, 1, 0, 0], 3) == 1 + 1
    assert sharding.converged_count([0, 1, 1, 1, 0, 0], 0) == 3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _shard_desc():
    return seeded(lambda: problems.config2(B=3, T=10), 2)  # 3 groups of 2: ranks get 2 groups and 1


def _worker(rank, world, port, out_dir):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "tests")]
    import torch.distributed as dist
    import oracle_lib
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    desc = _shard_desc()
    mine = sharding.shard(desc, rank, world)
    r = oracle_lib.solve_batch(mine, n_threads=1)
    local = {k: r[k] for k in ("x", "status", "total_cost", "n_qp_solves")}
    full = sharding.gather_results(local, desc.B, dist, group_size=desc.c.group_size)
    conv, _ = sharding.reduce_report(sharding.converged_count(r["status"], mine.c.group_size), 1.0, dist)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), conv=conv, B=mine.B, G=mine.c.group_size, **full)
    dist.destroy_process_group()


def test_two_rank_gloo_never_splits_a_group(oracle, tmp_path):
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    desc = _shard_desc()
    ref = oracle.solve_batch(desc, n_threads=1)
    sizes = []
    for rank in range(world):
        got = np.load(tmp_path / f"rank{rank}.npz")
        sizes.append(int(got["B"]))
        assert int(got["G"]) == 2
        for k in ("x", "status", "total_cost", "n_qp_solves"):
            np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
        assert got["conv"] == sharding.converged_count(ref["status"], 2)  # problems, not trajectories
    assert sizes == [4, 2]


def _write_input(path, d):
    robot = d.robot_spec
    names = [f"link{i}" for i in range(len(robot["segments"]))]
    with open(path, "w") as f:
        f.write(f"{d.B} {d.T} {d.D} {len(robot['segments'])} {d.c.group_size} {d.c.group_stop}\n")
        for i, s in enumerate(robot["segments"]):
            vals = [s.parent, s.joint_type, s.q_index, *s.origin_xyz, *s.origin_wxyz, *s.axis]
            f.write(" ".join(repr(float(v)) if isinstance(v, float) else str(v) for v in vals) + f" {names[i]}\n")
        f.write(" ".join(repr(float(v)) for v in robot["lower"]) + "\n")
        f.write(" ".join(repr(float(v)) for v in robot["upper"]) + "\n")
        f.write(f"{len(robot['spheres'])}\n")
        for sp in robot["spheres"]:
            f.write(f"{names[sp.segment]} " + " ".join(repr(float(v)) for v in (*sp.center, sp.radius)) + "\n")
        f.write(names[robot["tool"]] + "\n")
        for arr in (d.init_traj, d.cart_targets.reshape(d.B, 7)):
            f.write(" ".join(repr(float(v)) for v in arr.ravel()) + "\n")
        f.write(f"{d.obstacles.shape[1]}\n" + " ".join(repr(float(v)) for v in d.obstacles.ravel()) + "\n")


def test_cpp_layer_flattens_the_groups(host_bin, tmp_path):
    d = seeded(lambda: problems.config2(B=3, T=10), 4, group_stop=1)
    path = str(tmp_path / "in.txt")
    _write_input(path, d)
    out = subprocess.run([host_bin, path, "dump"], check=True, capture_output=True, text=True).stdout.split()
    assert out == ["batch", "12", "group_size", "4", "group_stop", "1"]


# --------------------------------------------------------------------------------------------------------------- GPU
def _device_solve(p, trace_cap=0):
    if trace_cap:
        p.lib.tb200_debug_enable_trace(p.handle, trace_cap)
    got = p.solve()
    B = p.desc.B
    if trace_cap:
        tr, tl = np.zeros((B, trace_cap, 14)), np.zeros(B, np.int32)
        p.lib.tb200_debug_fetch_trace(p.handle, tr.ctypes.data_as(_dbl_p), tl.ctypes.data_as(_i32_p))
        got["trace"], got["trace_len"] = tr, tl
    got["groups"] = p.group_results()
    done = np.zeros(B // p.group_size, np.int32)
    assert p.lib.tb200_debug_group_done(p.handle, done.ctypes.data_as(_i32_p)) == 0
    got["group_done"] = done
    return got


def _status_rule(cnt_viols, tol):
    return np.where(cnt_viols.max(axis=-1) < tol, capi.OPT_CONVERGED, capi.OPT_TIME_LIMIT)


def _check_selection(got, G):
    best, n_conv = select_cpu(got["status"], got["cnt_viols"], got["total_cost"], G)
    g = got["groups"]
    np.testing.assert_array_equal(g["best"], best)
    np.testing.assert_array_equal(g["n_converged"], n_conv)
    np.testing.assert_array_equal(g["status"], got["status"][best])
    assert g["total_cost"].tobytes() == got["total_cost"][best].tobytes()
    assert g["x"].tobytes() == got["x"][best].tobytes()


def _unverified(tr, tl, qp_max_iter):
    """A QP that hit the iteration limit or ended without a KKT-verified polish makes a trajectory incomparable with
    the CPU model step by step (tests/test_time_limit.py)."""
    return np.array([(tr[b, :tl[b], 7] >= qp_max_iter).any() or (tr[b, :tl[b], 12] != 1).any() for b in range(len(tl))])


CASES = {"cfg2_G8": lambda: cfg2_seeded(8), "cfg3_G4": lambda: cfg3_seeded(4)}


@pytest.fixture(scope="module")
def runs():
    """Per case: the ungrouped solve, group_stop 0 and group_stop 1 of the same batch, with decision traces."""
    out = {}
    for name, make in CASES.items():
        d = make()
        G = d.c.group_size
        d.c.group_size, d.c.group_stop = 0, 0
        p = api.Problem(d)
        plain = _device_solve(p, 600)
        p.set_groups(G, 0)
        stop0 = _device_solve(p, 600)
        p.set_groups(G, 1)
        stop1 = _device_solve(p, 600)
        p.close()
        out[name] = (d, G, plain, stop0, stop1)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_stop0_is_the_ungrouped_solve_plus_the_selection(runs, name):
    d, G, plain, stop0, _ = runs[name]
    for k in RESULT_KEYS + ("trace", "trace_len"):
        assert stop0[k].tobytes() == plain[k].tobytes(), k
    assert (stop0["groups"]["ended_by"] == 0).all() and (stop0["group_done"] == 0).all()
    _check_selection(stop0, G)
    # without groups every trajectory is its own group
    np.testing.assert_array_equal(plain["groups"]["best"], np.arange(d.B))
    _check_selection(plain, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_stop1_ends_siblings_of_a_converged_seed(runs, oracle, name):
    d, G, _, ref, got = runs[name]
    ended = got["groups"]["ended_by"]
    own, cut = ended == 0, ended == 2
    assert set(np.unique(ended)) <= {0, 2}
    assert cut.any() and own.any(), np.bincount(ended)
    # the trajectories that ended by their own SQP are bitwise the stop-0 ones
    for k in RESULT_KEYS:
        assert got[k][own].tobytes() == ref[k][own].tobytes(), k
    # a group-stopped seed has a sibling that converged by its own SQP, and its group's flag is set
    conv_own = (own & (got["status"] == capi.OPT_CONVERGED)).reshape(-1, G)
    grp = np.arange(d.B) // G
    assert conv_own.any(axis=1)[grp[cut]].all()
    np.testing.assert_array_equal(got["group_done"], conv_own.any(axis=1).astype(np.int32))
    # its decisions are a bitwise prefix of its stop-0 decisions, ending at an iteration top
    tf, lf, tl, ll = ref["trace"], ref["trace_len"], got["trace"], got["trace_len"]
    for b in np.nonzero(cut)[0]:
        n = ll[b]
        assert n < lf[b]
        assert tl[b, :n].tobytes() == tf[b, :n].tobytes(), b
        assert n == 0 or tuple(tf[b, n, :2]) != tuple(tf[b, n - 1, :2]), (b, tf[b, max(n - 1, 0):n + 1, :2])
    np.testing.assert_array_equal(got["n_qp_solves"][cut], ll[cut])
    np.testing.assert_array_equal(got["status"][cut], _status_rule(got["cnt_viols"][cut], d.c.sqp.cnt_tolerance))
    # a stopped seed against the CPU model with the device's QP counts as budgets, where every QP was KKT-verified (the
    # seeds that ended by their own SQP are the stop-0 results, bit for bit)
    ok = ~_unverified(tl, ll, d.c.qp.max_iter) & cut
    assert ok.sum() >= 0.75 * cut.sum()
    model = oracle.solve_batch(d, qp_budget=got["n_qp_solves"])
    np.testing.assert_array_equal(got["status"][ok], model["status"][ok])
    np.testing.assert_array_equal(got["n_qp_solves"][ok], model["n_qp_solves"][ok])
    np.testing.assert_allclose(got["total_cost"][ok], model["total_cost"][ok], atol=1e-6)
    np.testing.assert_array_equal(model["ended"][ok], 1)
    _check_selection(got, G)
    assert got["timing"]["total_ms"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_stop_keeps_the_solved_problems(runs, name):
    _, _, _, ref, got = runs[name]
    np.testing.assert_array_equal(got["groups"]["n_converged"] > 0, ref["groups"]["n_converged"] > 0)


@pytest.mark.gpu
def test_device_no_groups_and_one_group():
    d = cfg2_seeded(8)
    d.c.group_size, d.c.group_stop = 0, 0
    p = api.Problem(d)
    base = p.solve()
    for G, stop in ((1, 1), (0, 1), (0, 0)):
        p.set_groups(G, stop)
        got = _device_solve(p)
        for k in RESULT_KEYS:
            assert got[k].tobytes() == base[k].tobytes(), (G, stop, k)
        assert (got["groups"]["ended_by"] == 0).all()
        np.testing.assert_array_equal(got["groups"]["best"], np.arange(d.B))
    for stop in (0, 1):  # G = B: one group
        p.set_groups(d.B, stop)
        got = _device_solve(p)
        _check_selection(got, d.B)
        assert got["groups"]["best"].shape == (1,)
        if stop:
            assert got["group_done"][0] == 1 and (got["groups"]["ended_by"] == 2).any()
    p.close()


@pytest.mark.gpu
def test_device_groups_with_a_time_limit(runs):
    """max_time at the median finish time of a group_stop run: both rules fire, each as it says.  (Which seeds a group
    stops depends on the order in which the device finishes them, so the comparison is with the group_stop 0 run.)"""
    d, G, _, ref, _ = runs["cfg2_G8"]
    p = api.Problem(d)
    p.set_groups(G, 1)
    start = C.c_uint64(0)
    _device_solve(p)
    ended_ns = np.zeros(1 + 2 * d.B, np.uint64)
    p.lib.tb200_debug_schedule(p.handle, ended_ns.ctypes.data_as(C.POINTER(C.c_uint64)))
    p.lib.tb200_debug_time_limit(p.handle, C.byref(start), np.zeros(d.B, np.int32).ctypes.data_as(_i32_p))
    finish_s = (ended_ns[1:1 + d.B].astype(np.int64) - np.int64(start.value)) * 1e-9
    sqp = capi.default_sqp_params()
    sqp.max_time = float(np.median(finish_s))
    p.set_sqp_params(sqp)
    lim = _device_solve(p, 600)
    p.close()
    ended = lim["groups"]["ended_by"]
    assert (ended == 1).any() and (ended == 2).any(), np.bincount(ended)
    for k in RESULT_KEYS:  # unstopped trajectories are the unlimited, ungrouped ones
        assert lim[k][ended == 0].tobytes() == ref[k][ended == 0].tobytes(), k
    grp = np.arange(d.B) // G
    conv_own = ((ended == 0) & (lim["status"] == capi.OPT_CONVERGED)).reshape(-1, G).any(axis=1)
    assert conv_own[grp[ended == 2]].all()
    stopped = ended > 0
    np.testing.assert_array_equal(lim["status"][stopped], _status_rule(lim["cnt_viols"][stopped], d.c.sqp.cnt_tolerance))
    tf, tl, ll = ref["trace"], lim["trace"], lim["trace_len"]
    for b in np.nonzero(stopped)[0]:
        assert tl[b, :ll[b]].tobytes() == tf[b, :ll[b]].tobytes(), b
    _check_selection(lim, G)


def _cpp_solve(host_bin, tmp_path, d):
    path = str(tmp_path / "in.txt")
    _write_input(path, d)
    out = subprocess.run([host_bin, path, "solve"], check=True, capture_output=True, text=True).stdout.splitlines()
    rows = [line.split() for line in out]
    assert len(rows) == d.B // d.c.group_size and all(v[0] == "problem" for v in rows)
    return [(int(v[1]), int(v[2]), float(v[3]), np.array(v[4:], int)) for v in rows]


@pytest.mark.gpu
def test_cpp_and_python_layers_pick_the_c_abi_winners(host_bin, tmp_path):
    d = seeded(lambda: problems.config2(B=6, T=30), 4)
    p = api.Problem(d)
    ref = _device_solve(p)
    p.close()
    g = ref["groups"]
    _check_selection(ref, 4)
    py = api.solve(d, group_size=4, group_stop=0)
    for k in ("best", "status", "n_converged", "total_cost", "x", "ended_by"):
        assert py["groups"][k].tobytes() == g[k].tobytes(), k
    for q, (best, status, cost, seeds) in enumerate(_cpp_solve(host_bin, tmp_path, d)):
        assert (best, status, cost) == (g["best"][q], g["status"][q], g["total_cost"][q])
        np.testing.assert_array_equal(seeds, ref["status"][4 * q:4 * q + 4])


@pytest.mark.gpu
def test_cpp_and_python_layers_with_group_stop(host_bin, tmp_path):
    """With group_stop the stopped seeds depend on the device's finishing order, so each layer's winners are checked
    against its own seeds: the Python layer's by the CPU selection, the C++ layer's for a consistent best seed."""
    d = seeded(lambda: problems.config2(B=6, T=30), 4, group_stop=1)
    py = api.solve(d, group_size=4, group_stop=1)
    _check_selection(py, 4)
    for q, (best, status, cost, seeds) in enumerate(_cpp_solve(host_bin, tmp_path, d)):
        assert 4 * q <= best < 4 * q + 4 and seeds[best - 4 * q] == status
        assert (status == capi.OPT_CONVERGED) == (seeds == capi.OPT_CONVERGED).any()
        np.testing.assert_array_equal(py["groups"]["n_converged"][q] > 0, (seeds == capi.OPT_CONVERGED).any())
