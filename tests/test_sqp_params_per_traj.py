"""Per-trajectory optimizer parameters (tb200_problem_desc.sqp_per_traj, tb200_problem_set_sqp_params_per_traj;
DESIGN.md sections 4.1 and 6).

Trajectory b runs under row b of the table, every field of tb200_sqp_params included, and gives exactly what it gives in a
uniform batch under that row: trajectories never interact except through group_stop, so the checks are bit for bit.
CPU: the ctypes mirror against the header, the exported symbol, flattening with a table, slicing and sharding, the sweep
builder and the C++ layer's rows.  GPU (-m gpu): a table of copies against no table, a mixed batch against one uniform
solve per set and the CPU oracle, deadlines, groups, the setters and the C++ layer."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpp_host
from trajopt_b200 import api, capi, problems, sharding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESULT_KEYS = ("x", "status", "total_cost", "cost_vals", "cnt_viols", "n_qp_solves", "n_func_evals", "n_admm_iters")
DBL_MAX = np.finfo(np.float64).max


def params(**kw):
    p = capi.default_sqp_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


# five parameter sets that exercise every branch of the decision step: trust box and its ratios, max_iter, the merit
# rules and cnt_tolerance
SETS = [params(),
        params(trust_box_size=0.02, trust_expand_ratio=2.0),
        params(trust_box_size=0.3, trust_shrink_ratio=0.5, max_iter=8),
        params(merit_coeff_increase_ratio=3.0, initial_merit_error_coeff=2.0, inflate_constraints_individually=0),
        params(cnt_tolerance=1e-2, max_merit_coeff_increases=2, improve_ratio_threshold=0.1)]


def fields(p):
    return tuple(getattr(p, k) for k, _ in capi.SqpParams._fields_)


def with_table(d, rows):
    """d with a per-trajectory table (rows: B SqpParams)."""
    per = bool(d.c.obstacles_per_traj)
    return capi.ProblemDesc(d.robot_spec, d.T, d.terms, d.init_traj, fixed_timesteps=d._fixed_t, fixed_dofs=d._fixed_d,
                            cart_targets=d.cart_targets, obstacles=d.obstacles, obstacles_per_traj=per, sqp=d.c.sqp,
                            qp=d.c.qp, group_size=d.c.group_size, group_stop=d.c.group_stop, sqp_per_traj=rows)


def subset(d, idx, sqp):
    """Trajectories idx of d as a batch of their own, under the uniform parameters sqp (for the CPU oracle)."""
    per = bool(d.c.obstacles_per_traj)
    return capi.ProblemDesc(d.robot_spec, d.T, d.terms, d.init_traj[idx], fixed_timesteps=d._fixed_t,
                            fixed_dofs=d._fixed_d, cart_targets=None if d.cart_targets is None else d.cart_targets[idx],
                            obstacles=d.obstacles[idx] if per else d.obstacles, obstacles_per_traj=per, sqp=sqp, qp=d.c.qp)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_ctypes_mirror_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "trajopt_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", offsetof(tb200_problem_desc, sqp_per_traj), '
                   'sizeof(tb200_problem_desc), sizeof(tb200_sqp_params)); return 0; }\n')
    exe = str(tmp_path / "layout")  # (a C compile of the header, not a tests/cpp program)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe, "-lm"], check=True)
    off, size, row = map(int, subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split())
    assert off == capi.ProblemDescC.sqp_per_traj.offset
    assert size == C.sizeof(capi.ProblemDescC)
    assert row == C.sizeof(capi.SqpParams)


def test_setter_is_exported():
    lib = capi.load_library()
    assert "tb200_problem_set_sqp_params_per_traj" in capi.EXPORTED_SYMBOLS
    assert hasattr(lib, "tb200_problem_set_sqp_params_per_traj")


def test_a_zeroed_description_has_no_table():
    assert not capi.ProblemDescC().sqp_per_traj
    assert not problems.config2(B=4, T=10).c.sqp_per_traj


def test_description_with_a_table_flattens_and_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    d = problems.config2(B=5, T=10)
    d = with_table(d, SETS)
    lib = capi.load_library()
    h = C.c_void_p()
    rc = lib.tb200_problem_create(C.byref(d.c), 0, C.byref(h))
    assert rc == capi.ERR_NO_DEVICE, lib.tb200_last_error()


def test_table_needs_one_row_per_trajectory():
    d = problems.config2(B=4, T=10)
    with pytest.raises(ValueError):
        with_table(d, SETS[:3])


def test_slice_and_shard_keep_the_rows():
    d = problems.config2(B=10, T=10)
    rows = [params(trust_box_size=0.01 * (b + 1), max_iter=b + 1) for b in range(10)]
    d = with_table(d, rows)
    s = d.slice(3, 7)
    assert s.B == 4 and [fields(r) for r in s.sqp_per_traj] == [fields(r) for r in rows[3:7]]
    assert C.addressof(s.c.sqp_per_traj.contents) == C.addressof(s.sqp_per_traj)
    got = []
    for rank in range(3):
        sh = sharding.shard(d, rank, 3)
        got += [fields(r) for r in sh.sqp_per_traj]
    assert got == [fields(r) for r in rows]
    assert d.slice(0, 10).c.sqp_per_traj and problems.config2(B=4, T=10).slice(0, 2).sqp_per_traj is None


def test_shards_of_groups_keep_the_rows():
    base = problems.config2(B=3, T=10)
    g = problems.with_seeds(base, 4, np.random.default_rng(3), 0.5)
    rows = [params(trust_box_size=0.05 + 0.01 * b) for b in range(g.B)]
    g = with_table(g, rows)
    bounds = [sharding.shard_bounds(g.B, r, 2, g.c.group_size) for r in range(2)]
    assert bounds == [(0, 8), (8, 12)]
    for r, (b0, b1) in enumerate(bounds):
        sh = sharding.shard(g, r, 2)
        assert sh.c.group_size == 4 and [fields(x) for x in sh.sqp_per_traj] == [fields(x) for x in rows[b0:b1]]
    with pytest.raises(ValueError):
        g.slice(2, 6)
    # with_seeds repeats a table with the trajectories
    t = problems.with_seeds(with_table(base, SETS[:3]), 2, np.random.default_rng(3), 0.5)
    assert [fields(x) for x in t.sqp_per_traj] == [fields(SETS[k]) for k in (0, 0, 1, 1, 2, 2)]


def test_sweep_shapes():
    d = problems.config2(B=6, T=10)
    sets = [params(trust_box_size=tb, trust_shrink_ratio=sh, trust_expand_ratio=ex) for tb, sh, ex in problems.CONFIG4_SWEEP]
    s, idx = problems.sweep(d, sets)
    K = len(sets)
    assert K == 24 and s.B == K * d.B and idx.shape == (K * d.B,)
    np.testing.assert_array_equal(idx, np.repeat(np.arange(K), d.B))
    np.testing.assert_array_equal(s.init_traj, np.tile(d.init_traj, (K, 1, 1)))
    np.testing.assert_array_equal(s.cart_targets, np.tile(d.cart_targets, (K, 1, 1)))
    np.testing.assert_array_equal(s.obstacles, np.tile(d.obstacles, (K, 1, 1)))
    assert all(fields(s.sqp_per_traj[b]) == fields(sets[idx[b]]) for b in range(s.B))
    assert fields(s.c.sqp) == fields(d.c.sqp)
    g = problems.with_seeds(d, 2, np.random.default_rng(1), 0.5)
    sg, _ = problems.sweep(g, sets[:3])
    assert sg.B == 36 and sg.c.group_size == 2
    with pytest.raises(ValueError):
        problems.sweep(d, [])


@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "sqp_params_per_traj_host")


def test_cpp_rows_are_checked_and_in_order(host_bin):
    out = subprocess.run([host_bin, "rows"], check=True, capture_output=True, text=True).stdout.splitlines()
    assert out[0].startswith("invalid_argument") and "3 entries for a batch of 4" in out[0]
    rows = [line.split()[1:] for line in out[1:]]
    assert len(rows) == 3
    for b, r in enumerate(rows):
        assert float(r[0]) == 0.1 * (b + 1) and int(r[1]) == 10 + b and float(r[2]) == 1e-3 * (b + 1)
        assert float(r[3]) == (-1.0 if b == 1 else DBL_MAX) and int(r[4]) == (b != 2) and float(r[5]) == 10.0


# ------------------------------------------------------------------------------------------------------------------ GPU
def _solve(p, log_cap=400):
    """Results and the SQP log (with the points) of one solve of the problem handle p."""
    p.set_sqp_log(log_cap, with_x=True)
    out = p.solve()
    out["sqp_log"] = p.sqp_log()
    out["ended_by"] = p.group_results()["ended_by"]
    return out


def _same(a, b, idx=None, log=True):
    """Bit-for-bit equality of the results (and SQP logs) of trajectories idx."""
    idx = np.arange(len(a["status"])) if idx is None else np.asarray(idx)
    for k in RESULT_KEYS + ("ended_by",):
        x, y = np.asarray(a[k])[idx], np.asarray(b[k])[idx]
        assert x.tobytes() == y.tobytes(), (k, idx[np.nonzero((x != y).reshape(len(idx), -1).any(axis=1))[0]])
    if log:
        for k, v in a["sqp_log"].items():
            assert np.asarray(v)[idx].tobytes() == np.asarray(b["sqp_log"][k])[idx].tobytes(), ("sqp_log", k)


def _cases():
    return {"cfg2": problems.config2(B=64, T=20), "cfg4": problems.config4(B=10, T=12)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_table_of_copies_equals_no_table(name):
    d = _cases()[name]
    ref = _solve(api.Problem(d))
    got = _solve(api.Problem(with_table(d, [d.c.sqp] * d.B)))
    _same(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_mixed_batch_equals_uniform_solves(oracle, name):
    d = _cases()[name]
    s = np.arange(d.B) % len(SETS)
    got = _solve(api.Problem(with_table(d, [SETS[k] for k in s])))
    p = api.Problem(d)
    for k, sp in enumerate(SETS):
        p.set_sqp_params(sp)
        _same(got, _solve(p), np.nonzero(s == k)[0])
    # a few trajectories per set against the CPU oracle under that set (tolerances of test_gpu_parity.py)
    for k, sp in enumerate(SETS):
        idx = np.nonzero(s == k)[0][:2]
        ref = oracle.solve_batch(subset(d, idx, sp))
        assert (got["status"][idx] == ref["status"]).all() and (got["n_qp_solves"][idx] == ref["n_qp_solves"]).all()
        np.testing.assert_allclose(got["total_cost"][idx], ref["total_cost"], atol=1e-6)
        np.testing.assert_allclose(got["x"][idx], ref["x"], atol=1e-5)


@pytest.mark.gpu
def test_deadlines_per_trajectory():
    d = problems.config2(B=64, T=20)
    # the -1 rows end at the first check, with the status their own cnt_tolerance gives at the start point: never
    # within -1, always within 1e3; the DBL_MAX rows run untimed (the batch runs the clock check for the others)
    tol = [-1.0, 1e3]
    rows = [params(max_time=-1.0, cnt_tolerance=tol[(b // 2) % 2]) if b % 2 else params() for b in range(d.B)]
    got = _solve(api.Problem(with_table(d, rows)))
    ref = _solve(api.Problem(d))
    dead, free = np.arange(1, d.B, 2), np.arange(0, d.B, 2)
    assert (got["n_qp_solves"][dead] == 0).all() and (got["ended_by"][dead] == 1).all()
    for b in dead:
        want = capi.OPT_CONVERGED if rows[b].cnt_tolerance > 0 else capi.OPT_TIME_LIMIT
        assert got["status"][b] == want, (b, got["cnt_viols"][b], rows[b].cnt_tolerance)
    np.testing.assert_array_equal(got["x"][dead], ref["sqp_log"]["new_x"][dead, 0])  # the start point
    _same(got, ref, free)


@pytest.mark.gpu
def test_groups_with_a_mixed_table():
    base = problems.config2(B=16, T=20)
    g = problems.with_seeds(base, 4, np.random.default_rng(5), 0.6)
    rows = [SETS[b % 4] for b in range(g.B)]  # every seed of a group under its own set: a parameter portfolio
    p = api.Problem(with_table(g, rows))
    p.set_groups(0)
    flat = _solve(p)
    p.set_groups(4, 0)
    grouped = _solve(p)
    _same(grouped, flat)
    p.set_groups(4, 1)
    stopped = _solve(p)
    own = np.nonzero(stopped["ended_by"] == 0)[0]
    _same(stopped, flat, own)
    assert (stopped["ended_by"][stopped["ended_by"] != 0] == 2).all()
    solved = lambda r: (np.asarray(r["status"]) == 0).reshape(-1, 4).any(axis=1)  # noqa: E731
    np.testing.assert_array_equal(solved(stopped), solved(flat))


@pytest.mark.gpu
def test_setters_replace_and_clear_the_table(host_bin, tmp_path):
    d = problems.config2(B=12, T=20)
    rows = [SETS[b % 3 + 1] for b in range(d.B)]
    p = api.Problem(d)
    base = _solve(p)
    p.set_sqp_params(rows)
    mixed = _solve(p)
    assert any((mixed[k] != base[k]).any() for k in ("n_qp_solves", "total_cost"))
    p.set_sqp_params([SETS[0]] * d.B)
    _same(_solve(p), base)
    p.set_sqp_params(rows)
    p.set_sqp_params(None)  # drops the table: the uniform parameters again
    _same(_solve(p), base)
    p.set_sqp_params(rows)
    p.set_sqp_params(SETS[0])  # a uniform setting drops the table too
    _same(_solve(p), base)
    with pytest.raises(ValueError):
        p.set_sqp_params(rows[:5])
    # created with the table: the same as the setter
    _same(_solve(api.Problem(with_table(d, rows))), mixed)
    # the C++ layer (problem b under its set_params(b % 4)) returns what the C ABI returns
    cpp_sets = [params(trust_box_size=t, trust_shrink_ratio=s, max_iter=m)
                for t, s, m in ((0.1, 0.1, 50), (0.02, 0.5, 8), (0.3, 0.1, 30), (0.05, 0.3, 50))]
    g = problems.with_seeds(problems.config2(B=3, T=20), 4, np.random.default_rng(2), 0.5)
    want = api.Problem(with_table(g, [cpp_sets[b % 4] for b in range(g.B)])).solve()
    out = subprocess.run([host_bin, "solve", cpp_host.write_problem(tmp_path / "in.txt", g), "4", str(g.c.group_size),
                          str(g.c.group_stop)], check=True, capture_output=True, text=True).stdout.splitlines()
    assert out[0] == "throws"
    trajs = [line.split()[1:] for line in out[1:1 + g.B]]
    for b, (st, cost, nqp, nfe) in enumerate(trajs):
        assert (int(st), float(cost), int(nqp), int(nfe)) == \
            (want["status"][b], want["total_cost"][b], want["n_qp_solves"][b], want["n_func_evals"][b])
    probs = [line.split()[1:] for line in out[1 + g.B:]]
    assert len(probs) == g.B // 4


@pytest.mark.gpu
def test_sweep_in_one_solve_equals_one_solve_per_point():
    """What scripts/param_sweep.py checks, on configs[2]: the 24 points of the trust-region sweep as one batch of 24 * B
    with the table, against one uniform solve of B per point.  (The table of a large batch is uploaded after the zero
    fills of creation: at this size a table zeroed behind the upload changes every trajectory.)"""
    d = problems.config2(B=64, T=20)
    sets = [params(trust_box_size=tb, trust_shrink_ratio=sh, trust_expand_ratio=ex) for tb, sh, ex in problems.CONFIG4_SWEEP]
    tiled, idx = problems.sweep(d, sets)
    got = api.solve(tiled)
    p = api.Problem(d)
    for k, sp in enumerate(sets):
        p.set_sqp_params(sp)
        ref = p.solve()
        for key in RESULT_KEYS:
            assert got[key][idx == k].tobytes() == ref[key].tobytes(), (k, key)
