"""The SQP iteration log (tb200_problem_set_sqp_log / tb200_fetch_sqp_log; DESIGN.md section 4.7) and what is built on
it: the replayed optimizer callbacks and the log_results files of the C++ layer (include/trajopt_b200.hpp).

CPU: the ABI mirror, the refusals that need no device, and the C++ replay and writers on a synthetic log
(tests/cpp/sqp_log_host.cpp) against Python formatting with the reference's printf formats.  GPU (-m gpu): logging
does not change a result bit, the records obey the SQP's own rules, agree with the decision trace and the CPU oracle,
truncate to a prefix, stop with the time limit and the group stop, and the C++ layer replays and writes them."""
import ctypes as C
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import cpp_host
from trajopt_b200 import api, capi, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_dbl_p = C.POINTER(C.c_double)
_i32_p = C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def host_bin(tmp_path_factory):
    return cpp_host.build(tmp_path_factory, "sqp_log_host")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_abi_struct_matches_header():
    """tb200_sqp_log is 23 pointers in header order; the new entry points are exported."""
    names = [n for n, _ in capi.SqpLog._fields_]
    assert C.sizeof(capi.SqpLog) == 23 * 8
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    body = hdr[hdr.index("typedef struct tb200_sqp_log {"):hdr.index("} tb200_sqp_log;")]
    fields = re.findall(r"^\s*(?:int32_t|double)\* (\w+);", body, re.M)
    assert fields == names
    for k, n in enumerate(names):
        assert getattr(capi.SqpLog, n).offset == 8 * k
    lib = capi.load_library()
    for s in ("tb200_problem_set_sqp_log", "tb200_fetch_sqp_log", "tb200_problem_objects"):
        assert s in capi.EXPORTED_SYMBOLS and hasattr(lib, s)
    assert "#define TB200_VERSION_MINOR 5" in hdr


def test_null_problem_is_refused():
    lib = capi.load_library()
    assert lib.tb200_problem_set_sqp_log(None, 4, 0) == capi.ERR_INVALID
    assert lib.tb200_fetch_sqp_log(None, C.byref(capi.SqpLog())) == capi.ERR_INVALID
    assert lib.tb200_problem_objects(None, None, None) == capi.ERR_INVALID


def _fmt_e(v):
    return "%e" % v


def _expected_files(recs, mu_of, names_c, names_k, var_names):
    """The reference's BasicTrustRegionSQPResults::write* (optimizers.cpp:533-647) in Python."""
    solver, vars_, costs, cnts = [], [], [], []
    for i, r in enumerate(recs):
        om, mm, nm = r["old_merit"], r["model_merit"], r["new_merit"]
        a, e = om - mm, om - nm
        if i == 0:
            solver.append("DESCRIPTION,oldexact,new_exact,dapprox,dexact,ratio")
            vars_.append("NAMES" + "".join("," + v for v in var_names))
            costs.append("COST NAMES" + "".join(",%s,%s,%s,%s" % (n, n, n, n) for n in names_c))
            costs.append("DESCRIPTION" + ",oldexact,dapprox,dexact,ratio" * len(names_c))
            cnts.append("CONSTRAINT NAMES" + "".join(",%s,%s,%s,%s" % (n, n, n, n) for n in names_k))
            cnts.append("DESCRIPTION" + ",oldexact,dapprox,dexact,ratio" * len(names_k))
        solver.append("%s,%10.3e,%10.3e,%10.3e,%10.3e,%10.3e" % ("Solver", om, nm, a, e, e / a))
        vars_.append("VALUES" + "".join("," + _fmt_e(v) for v in r["x"]))
        line = "COSTS"
        for o, m, w in zip(r["oc"], r["mc"], r["nc"]):
            a, e = o - m, o - w
            line += ",%e,%e,%e,%e" % (o, a, e, e / a) if abs(a) > 1e-8 else ",%e,%e,%e,%s" % (o, a, e, "nan")
        costs.append(line)
        line = "CONSTRAINTS"
        for o, m, w, mu in zip(r["ok"], r["mk"], r["nk"], r["mu"]):
            a, e = o - m, o - w
            line += (",%e,%e,%e,%e" % (mu * o, mu * a, mu * e, e / a) if abs(a) > 1e-8
                     else ",%e,%e,%e,%s" % (mu * o, mu * a, mu * e, "nan"))
        cnts.append(line)
    return {"trajopt_solver.log": solver, "trajopt_vars.log": vars_, "trajopt_costs.log": costs,
            "trajopt_constraints.log": cnts}


# the synthetic log of sqp_log_host.cpp: (kind, round, iter, action, mu, mc, mk, nc, nk, x0, x1) per record
_SYN = {0: [(0, 0, 1, -1, 10, None, None, 5.0, 0.5, 0.1, 0.2), (1, 0, 1, 3, 10, None, None, None, None, None, None),
            (1, 0, 1, 0, 10, 1.0, 0.1, 7.0, 0.4, 0.3, 0.3), (1, 0, 1, 1, 10, 3.0, 0.2, 4.0, 0.25, 0.15, 0.25),
            (1, 0, 2, 1, 10, 2.5, 0.1, 3.5, 0.125, 0.175, 0.3), (1, 0, 3, 2, 10, 3.4999999999, 0.125, 3.5, 0.125, 0.175, 0.3)],
        1: [(0, 0, 1, -1, 10, None, None, 1.0, 2.0, -0.5, 0.5), (1, 0, 1, 1, 10, 0.5, 1.0, 0.75, 1.5, -0.25, 0.5),
            (1, 0, 2, 0, 10, 0.5, 1.0, 0.8, 1.6, -0.2, 0.4), (1, 1, 1, 1, 100, 0.5, 0.5, 0.6, 0.75, -0.1, 0.3)]}


def _syn_records(recs):
    """Successful QP records with the derived old values and merits, as the fetch fills them."""
    out, last = [], recs[0]
    for r in recs[1:]:
        kind, rnd, it, act, mu, mc, mk, nc, nk, x0, x1 = r
        if act != 3:
            oc, ok = last[7], last[8]
            out.append(dict(old_merit=oc + ok * mu, model_merit=mc + mk * mu, new_merit=nc + nk * mu, x=[x0, x1],
                            oc=[oc], mc=[mc], nc=[nc], ok=[ok], mk=[mk], nk=[nk], mu=[mu]))
        if act == 1:
            last = r
    return out


def test_cpp_replay_and_writers_on_a_synthetic_log(host_bin, tmp_path):
    out = subprocess.run([host_bin, "synth", str(tmp_path)], check=True, capture_output=True, text=True).stdout.splitlines()
    cbs = [line.split() for line in out if line.startswith("cb ")]
    # problem 0: tops (0,1), (0,2), (0,3), then the final call; problem 1 (two records dropped, replayed as allowed):
    # tops (0,1), (0,2), (1,1), final
    got = [(int(v[1]), int(v[3]), int(v[4]), int(v[7]), int(v[8])) for v in cbs]  # problem, n_qp, n_fe, |cost|, |cnt|
    assert got == [(0, 0, 0, 0, 0), (0, 3, 3, 1, 1), (0, 4, 4, 1, 1), (0, 99, 0, 0, 0),
                   (1, 0, 0, 0, 0), (1, 1, 2, 1, 1), (1, 2, 3, 1, 1), (1, 99, 0, 0, 0)]
    # x: the start point at the first top, then the last accepted point
    xs = [[float(t) for t in v[9:11]] for v in cbs if int(v[6]) == 2]
    assert xs == [[0.1, 0.2], [0.15, 0.25], [0.175, 0.3], [-0.5, 0.5], [-0.25, 0.5], [-0.25, 0.5]]
    assert [float(t) for t in cbs[1][11:13]] == [4.0, 0.25]  # the accepted point's exact values
    assert any(line.startswith("refused SQP log of problem 1 is truncated") for line in out)
    for b in (0, 1):
        want = _expected_files(_syn_records(_SYN[b]), None, ["joint_vel"], ["collision_3"], ["j_0_0", "j_0_1"])
        for name, lines in want.items():
            assert open(tmp_path / str(b) / name).read() == "".join(line + "\n" for line in lines), (b, name)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _solve(d, cap=0, with_x=False):
    p = api.Problem(d)
    try:
        if cap:
            p.set_sqp_log(cap, with_x)
        out = p.solve()
        if cap:
            out["log"] = p.sqp_log()
        return out
    finally:
        p.close()


_RESULT_KEYS = ("x", "status", "total_cost", "cost_vals", "cnt_viols", "n_qp_solves", "n_func_evals", "n_admm_iters")
_CASES = {"cfg1": lambda: problems.config1(B=16, T=12), "cfg2": lambda: problems.config2(B=32, T=30),
          "cfg4": lambda: problems.config4(B=8, T=12), "cfg3": lambda: problems.config3(B=8, T=30)}


def _same_results(a, b):
    for k in _RESULT_KEYS:
        assert a[k].tobytes() == b[k].tobytes(), k


def _fma(a, b, c):
    """a * b + c rounded once, as the device's contracted multiply-add"""
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _merit(v, nk_vals, mu):
    """The device's merit: the costs summed in order, plus the violations times their coefficients in order."""
    s = 0.0
    for c in v:
        s += c
    t = 0.0
    for k, m in zip(nk_vals, mu):
        t = _fma(k, m, t)
    return s + t


@pytest.fixture(scope="module")
def runs():
    out = {}
    for name, make in _CASES.items():
        d = make()
        out[name] = (d, _solve(d), _solve(d, 400, True))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_log_does_not_change_results(runs, name):
    d, off, on = runs[name]
    _same_results(off, on)


@pytest.mark.gpu
def test_handle_with_log_disabled_again_solves_as_before(runs):
    d, off, _ = runs["cfg2"]
    p = api.Problem(d)
    try:
        p.set_sqp_log(50, True)
        p.solve()
        p.set_sqp_log(0)
        _same_results(off, p.solve())
        with pytest.raises(RuntimeError, match="without the SQP log"):
            p.sqp_log()
        with pytest.raises(RuntimeError, match="capacity"):
            p.set_sqp_log(-1)
        with pytest.raises(RuntimeError, match="with_x"):
            p.lib and p._check(p.lib.tb200_problem_set_sqp_log(p.handle, 4, 2))
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_records_obey_the_sqp(runs, name):
    d, off, on = runs[name]
    L, s = on["log"], d.c.sqp
    nr = L["n_records"]
    assert (L["n_dropped"] == 0).all()
    np.testing.assert_array_equal(nr, off["n_qp_solves"] + 1)
    for b in range(d.B):
        n = nr[b]
        kind, act = L["kind"][b, :n], L["action"][b, :n]
        assert kind[0] == 0 and (kind[1:] == 1).all()
        assert (L["ended"][b, :n - 1] == -1).all() and L["ended"][b, n - 1] == off["status"][b]
        # the last accepted record (or kind 0) holds the results
        last = ([0] + [r for r in range(1, n) if act[r] == 1])[-1]
        assert L["new_x"][b, last].tobytes() == off["x"][b].tobytes()
        assert L["new_cost_vals"][b, last].tobytes() == off["cost_vals"][b].tobytes()
        assert L["new_cnt_viols"][b, last].tobytes() == off["cnt_viols"][b].tobytes()
        assert L["trust_box_size"][b, 0] == s.trust_box_size
        for r in range(1, n):
            mu = L["merit_coeffs"][b, r]
            if act[r] != 3:  # the merits are the device's in-order sums of the logged arrays
                assert L["old_merit"][b, r] == _merit(L["old_cost_vals"][b, r], L["old_cnt_viols"][b, r], mu)
                assert L["model_merit"][b, r] == _merit(L["model_cost_vals"][b, r], L["model_cnt_viols"][b, r], mu)
                assert L["new_merit"][b, r] == _merit(L["new_cost_vals"][b, r], L["new_cnt_viols"][b, r], mu)
            else:
                assert np.isnan(L["new_merit"][b, r]) and np.isnan(L["new_x"][b, r]).all()
            prev_mu = L["merit_coeffs"][b, r - 1]
            if L["merit_round"][b, r] == L["merit_round"][b, r - 1]:
                assert mu.tobytes() == prev_mu.tobytes()
            else:  # a penalty round: inflated by the ratio (all, or the violated ones)
                assert L["merit_round"][b, r] == L["merit_round"][b, r - 1] + 1 and L["iter"][b, r] == 1
                assert np.all((mu == prev_mu * s.merit_coeff_increase_ratio) | (mu == prev_mu))
            if r >= 2:  # the trust box follows from the previous record's action
                t0, a0 = L["trust_box_size"][b, r - 1], act[r - 1]
                t = L["trust_box_size"][b, r]
                if L["merit_round"][b, r] != L["merit_round"][b, r - 1]:
                    base = t0 * s.trust_expand_ratio if a0 == 1 else (t0 * s.trust_shrink_ratio if a0 == 0 else t0)
                    assert t == max(base, s.min_trust_box_size / s.trust_shrink_ratio * 1.5)
                elif a0 == 1:
                    assert t == t0 * s.trust_expand_ratio
                elif a0 == 0:
                    assert t == t0 * s.trust_shrink_ratio
                elif a0 == 3:
                    assert t in (t0 * s.trust_shrink_ratio, s.min_trust_box_size)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_log_equals_the_decision_trace(runs, name):
    d, _, _ = runs[name]
    p = api.Problem(d)
    try:
        cap = 400
        p.lib.tb200_debug_enable_trace(p.handle, cap)
        p.set_sqp_log(cap + 1, False)
        p.solve()
        tr, tl = np.zeros((d.B, cap, 14)), np.zeros(d.B, np.int32)
        p.lib.tb200_debug_fetch_trace(p.handle, tr.ctypes.data_as(_dbl_p), tl.ctypes.data_as(_i32_p))
        L = p.sqp_log()
    finally:
        p.close()
    np.testing.assert_array_equal(tl + 1, L["n_records"])
    for b in range(d.B):
        n = tl[b]
        t = tr[b, :n]
        sl = slice(1, n + 1)
        ok = L["action"][b, sl] != 3
        cols = [L["merit_round"][b, sl], L["iter"][b, sl], L["trust_box_size"][b, sl],
                np.where(ok, L["old_merit"][b, sl], 0.0), np.where(ok, L["model_merit"][b, sl], 0.0),
                np.where(ok, L["new_merit"][b, sl], 0.0), L["qp_status"][b, sl], L["admm_iters"][b, sl],
                L["action"][b, sl], L["qp_diag"][b, sl, 0], L["qp_diag"][b, sl, 1], L["qp_diag"][b, sl, 2],
                L["polish"][b, sl], L["qp_diag"][b, sl, 3]]
        assert np.stack([np.asarray(c, np.float64) for c in cols], 1).tobytes() == t.tobytes(), b


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_CASES))
def test_log_against_the_cpu_oracle(oracle, runs, name):
    """The oracle's decision trace of every trajectory against the log: the same decisions; values to 1e-8 (configs[3]:
    the loose rule of test_gpu_parity - its long QPs may stop on a different ADMM check, so only the final status and a
    shared prefix are compared)."""
    d, off, on = runs[name]
    L = on["log"]
    loose = name == "cfg3"
    for b in range(d.B):
        ref = oracle.solve_batch(d, b0=b, b1=b + 1, trace_b=b)["trace"]
        n = L["n_records"][b] - 1
        sl = slice(1, n + 1)
        dev = np.stack([L["merit_round"][b, sl], L["iter"][b, sl], L["action"][b, sl]], 1)
        if loose:
            m = min(len(ref), n, 3)
            np.testing.assert_array_equal(dev[:m], ref[:m, [0, 1, 8]])
            continue
        assert len(ref) == n, b
        np.testing.assert_array_equal(dev, ref[:, [0, 1, 8]])
        np.testing.assert_array_equal((L["qp_status"][b, sl] == 1) | (L["qp_status"][b, sl] == 2), ref[:, 6] == 1)
        ok = L["action"][b, sl] != 3
        for c, k in ((2, "trust_box_size"), (3, "old_merit"), (4, "model_merit"), (5, "new_merit")):
            v = L[k][b, sl]
            np.testing.assert_allclose(v[ok] if c > 2 else v, ref[ok, c] if c > 2 else ref[:, c], rtol=1e-8, atol=1e-8)


@pytest.mark.gpu
def test_truncation_keeps_the_prefix(runs):
    d, off, on = runs["cfg2"]
    full = on["log"]
    p = api.Problem(d)
    try:
        p.set_sqp_log(5, True)
        _same_results(off, p.solve())
        small = p.sqp_log()
    finally:
        p.close()
    np.testing.assert_array_equal(small["n_records"], np.minimum(full["n_records"], 5))
    np.testing.assert_array_equal(small["n_dropped"], np.maximum(full["n_records"] - 5, 0))
    for k, v in small.items():
        if v.ndim >= 2:
            assert v.tobytes() == np.ascontiguousarray(full[k][:, :5]).tobytes(), k


@pytest.mark.gpu
def test_time_limit_zero_leaves_the_initial_record():
    d = problems.config2(B=8, T=12)
    d.c.sqp.max_time = 0.0
    out = api.solve(d, sqp_log=8)
    L = out["sqp_log"]
    np.testing.assert_array_equal(L["n_records"], 1)
    assert (L["kind"][:, 0] == 0).all() and (L["ended"][:, 0] == -1).all()
    assert out["cost_vals"].tobytes() == np.ascontiguousarray(L["new_cost_vals"][:, 0]).tobytes()


@pytest.mark.gpu
def test_group_stop_ends_the_stopped_seeds_logs():
    d = problems.with_seeds(problems.config2(B=8, T=30), 4, np.random.default_rng(7), 0.6, group_stop=1)
    p = api.Problem(d)
    try:
        p.set_sqp_log(400, False)
        out = p.solve()
        L = p.sqp_log()
        ended = p.group_results()["ended_by"]
    finally:
        p.close()
    np.testing.assert_array_equal(L["n_records"], out["n_qp_solves"] + 1)
    for b in np.nonzero(ended == 2)[0]:
        n = L["n_records"][b]
        assert L["ended"][b, n - 1] == -1  # its last record is its last QP; the stop came at the next iteration top


@pytest.mark.gpu
def test_cpp_callbacks_and_log_results(host_bin, tmp_path):
    d = problems.config2(B=4, T=12)
    out = subprocess.run([host_bin, "solve", cpp_host.write_problem(tmp_path / "in.txt", d), str(tmp_path / "logs")],
                         check=True, capture_output=True, text=True).stdout.splitlines()
    rows = [line.split() for line in out]
    final = {int(v[1]): v[2:] for v in rows if v[0] == "final"}
    plain = {int(v[1]): v[2:] for v in rows if v[0] == "plain"}
    assert final == plain  # the logged solve returns the plain solve's results
    p = api.Problem(d)
    try:
        p.set_sqp_log(256, True)
        p.solve()
        L = p.sqp_log()
        term, step = p.objects()
    finally:
        p.close()
    for b in range(d.B):
        cbs = [v for v in rows if v[0] == "cb" and int(v[1]) == b]
        n = L["n_records"][b]
        tops = {(L["merit_round"][b, r], L["iter"][b, r]) for r in range(1, n)}
        assert len(cbs) == len(tops) + 1 and cbs[-1][2:] == final[b]
        assert cbs[0][3:5] == ["0", "0"]
        # the log_results files parse back to the log
        ok = [r for r in range(1, n) if L["action"][b, r] != 3]
        lines = open(tmp_path / "logs" / str(b) / "trajopt_vars.log").read().splitlines()
        assert lines[0] == "NAMES," + ",".join(f"j_{t}_{j}" for t in range(d.T) for j in range(d.D))
        vals = np.array([[float(t) for t in line.split(",")[1:]] for line in lines[1:]])
        np.testing.assert_allclose(vals, L["new_x"][b, ok].reshape(len(ok), -1), rtol=1e-6, atol=1e-300)
        solver = open(tmp_path / "logs" / str(b) / "trajopt_solver.log").read().splitlines()[1:]
        sv = np.array([[float(t) for t in line.split(",")[1:3]] for line in solver])
        np.testing.assert_allclose(sv, np.stack([L["old_merit"][b, ok], L["new_merit"][b, ok]], 1), rtol=1e-3)
    assert len(term) == len(step) == p.layout.n_costs + p.layout.n_cnts
    # object names as the reference's hatch forms them, in both files of every problem
    names_c = ["joint_vel", "joint_acc"]
    names_k = ["cart_pose"] + [f"collision_{t}" for t in range(1, d.T)]
    for b in range(d.B):
        for f, title, nm in (("trajopt_costs.log", "COST NAMES", names_c), ("trajopt_constraints.log", "CONSTRAINT NAMES", names_k)):
            first = open(tmp_path / "logs" / str(b) / f).readline().rstrip("\n")
            assert first == title + "".join(",%s,%s,%s,%s" % (n, n, n, n) for n in nm)
    # WriteCallback beside it: the header, then per callback T waypoint lines and an empty line
    csv = open(tmp_path / "logs" / "write.csv").read().split("\n")
    assert csv[0].endswith(",x,y,z,q_w,q_x,q_y,q_z," + ",".join(names_c + names_k))
    n_cb = sum(1 for v in rows if v[0] == "cb")
    assert len(csv) == 1 + n_cb * (d.T + 1) + 1 and csv[-1] == ""


_SMALL = {"cfg1": lambda: problems.config1(B=4, T=12), "cfg2": lambda: problems.config2(B=4, T=12),
          "cfg4": lambda: problems.config4(B=2, T=12)}


@pytest.mark.parametrize("name", list(_SMALL))
def test_log_model_is_the_oracle_driver(oracle, name):
    """With records on, the oracle's final results are those with records off, bit for bit, and its records' 14 trace
    columns are the oracle's TraceEntry list; record 0 is the clamped start with its exact values."""
    d = _SMALL[name]()
    got = oracle.solve_batch(d, records=512)
    ref = oracle.solve_batch(d)
    for k in ("x", "status", "total_cost", "cost_vals", "cnt_viols", "n_qp_solves", "n_func_evals", "n_admm_iters"):
        assert got[k].tobytes() == ref[k].tobytes(), k
    L = got["log"]
    np.testing.assert_array_equal(L["n_records"], ref["n_qp_solves"] + 1)
    for b in range(d.B):
        tr = oracle.solve_batch(d, b0=b, b1=b + 1, trace_b=b)["trace"]
        n = L["n_records"][b]
        assert L["trace"][b, 1:n].tobytes() == tr.tobytes(), b
        assert L["mu"][b, 0].tobytes() == np.full(L["mu"].shape[2], d.c.sqp.initial_merit_error_coeff).tobytes()
    # the accepted records' exact values chain into the final results
    for b in range(d.B):
        n = L["n_records"][b]
        acc = [0] + [r for r in range(1, n) if L["trace"][b, r, 8] == 1]
        assert L["new_cost_vals"][b, acc[-1]].tobytes() == ref["cost_vals"][b].tobytes()
        assert L["x"][b, acc[-1]].tobytes() == ref["x"][b].ravel().tobytes()


@pytest.mark.parametrize("make", [lambda: problems.config2(B=1, T=12), lambda: problems.config4(B=1, T=6)])
def test_host_fk_is_the_oracle_fk(oracle, host_bin, tmp_path, make):
    """RobotFK of the C++ header restates the oracle's Robot::fk: the same frames, to the last bits."""
    d = make()
    out = subprocess.run([host_bin, "fk", cpp_host.write_problem(tmp_path / "in.txt", d)], check=True,
                         capture_output=True, text=True).stdout.splitlines()
    S = len(d.robot_spec["segments"])
    got = np.array([[float(t) for t in line.split()[3:]] for line in out]).reshape(d.T, S, 12)
    for t in range(d.T):
        fr = np.zeros((S, 12))
        assert oracle.lib().oracle_fk(C.byref(d.c.robot), d.init_traj[0, t].ctypes.data_as(_dbl_p),
                                      fr.ctypes.data_as(_dbl_p)) == 0
        # (the oracle is built with FMA contraction, -march=x86-64-v3, the test program without: last bits differ)
        np.testing.assert_allclose(got[t], fr, rtol=0, atol=1e-14, err_msg=str(t))


def _quat_wxyz(m):
    """Eigen::Quaterniond(Matrix3d), row-major m: the trace branch and the largest-diagonal branch."""
    q = [0.0] * 4
    t = m[0] + m[4] + m[8]
    if t > 0:
        t = np.sqrt(t + 1.0)
        q[0] = 0.5 * t
        t = 0.5 / t
        q[1], q[2], q[3] = (m[7] - m[5]) * t, (m[2] - m[6]) * t, (m[3] - m[1]) * t
    else:
        i = 0
        if m[4] > m[0]:
            i = 1
        if m[8] > m[i * 3 + i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0)
        q[1 + i] = 0.5 * t
        t = 0.5 / t
        q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t
        q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t
        q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t
    return q


def test_write_callback_csv_layout(oracle, host_bin, tmp_path):
    """WriteCallback writes file_write_callback.cpp's layout: a header of joint names, x..q_z and the object names; per
    call one line per waypoint (joint values, then "<link>: " and the pose of every link, then the costs and the
    constraint values), and an empty line; numbers as operator<< prints them (%g)."""
    d = problems.config2(B=1, T=5)
    csv = str(tmp_path / "w.csv")
    subprocess.run([host_bin, "write", cpp_host.write_problem(tmp_path / "in.txt", d), csv], check=True)
    segs = d.robot_spec["segments"]
    names = [f"link{i}" for i in range(len(segs))]
    cols = {s.q_index: names[i] for i, s in enumerate(segs) if s.joint_type != capi.JOINT_FIXED}
    head = ",".join(cols[j] for j in range(d.D)) + ",x,y,z,q_w,q_x,q_y,q_z,joint_vel,joint_acc,cart_pose,collision_3"
    block = []
    for t in range(d.T):
        q = d.init_traj[0, t]
        fr = np.zeros((len(segs), 12))
        oracle.lib().oracle_fk(C.byref(d.c.robot), q.ctypes.data_as(_dbl_p), fr.ctypes.data_as(_dbl_p))
        line = ",".join("%g" % v for v in q)
        for s in sorted(range(len(segs)), key=lambda i: names[i]):
            line += names[s] + ": " + "".join(",%g" % v for v in [*fr[s, 9:], *_quat_wxyz(fr[s, :9])])
        block.append(line)
    want = [head]
    for c0 in (1.5, 3.0):
        want += [line + ",%g,%g,%g,%g" % (c0, 0.0625, 0.25, 1e-7) for line in block] + [""]
    assert open(csv).read() == "".join(line + "\n" for line in want)


def _expected_objects(d):
    """(term, step) of every object in OptProb order (costs, EQ constraints, INEQ constraints), from the description
    the way TermInfo::hatch makes them."""
    costs, eqs, ineqs = [], [], []
    for k, t in enumerate(d.terms):
        cnt = t.role == capi.ROLE_CNT
        if t.kind in (capi.TERM_JOINT_POS, capi.TERM_JOINT_VEL, capi.TERM_JOINT_ACC):
            eq = all(abs(t.upper_tols[j]) < 1e-5 and abs(t.lower_tols[j]) < 1e-5 for j in range(d.D))
            (costs if not cnt else (eqs if eq else ineqs)).append((k, t.first_step))
        elif t.kind == capi.TERM_CART_POSE:
            (eqs if cnt else costs).append((k, t.first_step))
        elif t.kind == capi.TERM_CART_VEL:
            for s in range(t.first_step, t.last_step + 1):
                (ineqs if cnt else costs).append((k, s))
        elif t.kind == capi.TERM_COLLISION:
            cast = t.evaluator_type != capi.COLL_DISCRETE
            fixed = set(t.fixed_steps[:t.n_fixed_steps])
            for s in range(t.first_step, t.last_step if cast else t.last_step + 1):
                if cast or s not in fixed:
                    (ineqs if cnt else costs).append((k, s))
    return costs + eqs + ineqs


@pytest.mark.gpu
@pytest.mark.parametrize("make", [lambda: problems.config2(B=2, T=12), lambda: problems.config3(B=2, T=12, via_every=4)])
def test_objects_name_their_terms_and_steps(make):
    d = make()
    p = api.Problem(d)
    try:
        term, step = p.objects()
        assert len(term) == p.layout.n_costs + p.layout.n_cnts
    finally:
        p.close()
    assert list(zip(term.tolist(), step.tolist())) == _expected_objects(d)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg1", "cfg2", "cfg4", "cfg3"])
def test_log_against_the_cpu_model(oracle, runs, name):
    """Every record of every trajectory against the CPU model of the log: the same count, kinds, (round, iter), actions
    and QP outcomes; merit coefficients, per-object model and exact values and the trust box within 1e-8; the points
    within the final-point rule of test_gpu_parity (1e-5).  configs[3]: the loose rule of test_gpu_parity - its long QPs
    may stop on a different ADMM check - so the decisions of a shared prefix only."""
    d, off, on = runs[name]
    L = on["log"]
    ref = oracle.solve_batch(d, records=512)["log"]
    for b in range(d.B):
        n = L["n_records"][b]
        if name == "cfg3":
            m = min(n, ref["n_records"][b], 4)
            np.testing.assert_array_equal(L["action"][b, 1:m], ref["trace"][b, 1:m, 8])
            continue
        assert n == ref["n_records"][b], b
        tr = ref["trace"][b, 1:n]
        np.testing.assert_array_equal(L["kind"][b, :n], [0] + [1] * (n - 1))
        np.testing.assert_array_equal(L["merit_round"][b, 1:n], tr[:, 0])
        np.testing.assert_array_equal(L["iter"][b, 1:n], tr[:, 1])
        np.testing.assert_array_equal(L["action"][b, 1:n], tr[:, 8])
        np.testing.assert_allclose(L["trust_box_size"][b, 1:n], tr[:, 2], rtol=1e-8, atol=1e-8)
        for k_dev, k_ref in (("merit_coeffs", "mu"), ("model_cost_vals", "model_cost_vals"),
                             ("model_cnt_viols", "model_cnt_viols"), ("new_cost_vals", "new_cost_vals"),
                             ("new_cnt_viols", "new_cnt_viols")):
            np.testing.assert_allclose(L[k_dev][b, :n], ref[k_ref][b, :n], rtol=1e-8, atol=1e-8, err_msg=f"{k_dev} {b}")
        np.testing.assert_allclose(L["new_x"][b, :n].reshape(n, -1), ref["x"][b, :n], atol=1e-5, err_msg=f"x {b}")
