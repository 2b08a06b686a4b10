"""GPU: the pose graph's ceres minimiser (include/d2pgo.h d2pgo_set_minimizer, D2PGO_MINIMIZER_CERES_LM) against its CPU oracle
(oracle/pgo_ceres_lm_oracle.py) iteration by iteration on 6-DoF, 4-DoF (yaws across +-pi), 6-DoF + gravity and the bench graph;
ARock local solves on it; the time budget; reproducibility; one host synchronisation per solve; refusals."""
import numpy as np
import pytest

from d2slam_b200 import pgo
from oracle import pgo_arock_oracle as ao
from oracle import pgo_ceres_lm_oracle as co
from oracle import pgo_lm_oracle as lo

import test_pgo_arock as tpa
import test_pgo_cholesky as tc

KINDS = {v: k for k, v in pgo.STEP_KINDS.items()}


def device(g, dof, ego=None, **cfg):
    s = tc.device(g, dof, ego)
    s.set_minimizer("ceres_lm", **cfg)
    return s


def poses(s, g, dof):
    return s.get_poses_4d(g["ids"]) if dof == 4 else s.get_poses(g["ids"])


def rotated_4d(seed):
    """a 4-DoF graph turned about z so that its yaws cross +-pi (relative measurements are unchanged)"""
    h = pgo.pose_graph_to_4d(tc.small_graph(seed=seed, n=40, loops=100), seed=seed)
    th = np.pi - float(np.median(h["init"][:, 3]))
    c, s_ = np.cos(th), np.sin(th)
    x = h["init"].copy()
    x[:, 0], x[:, 1] = c * h["init"][:, 0] - s_ * h["init"][:, 1], s_ * h["init"][:, 0] + c * h["init"][:, 1]
    x[:, 3] = pgo.normalize_angle(x[:, 3] + th)
    assert (x[:, 3] > 3.0).any() and (x[:, 3] < -3.0).any()
    return dict(h, init=x)


def case(name):
    if name == "4dof":
        h = rotated_4d(12)
        return h, 4, None, lo.Problem(h["init"], h["fixed"], h["ea"], h["eb"], h["rel"], h["sqrt_info"])
    if name == "bench":
        g = pgo.make_pose_graph(seed=7, n_agents=8, poses_per_agent=1250, loops=30001)
        prob, g, ego = tc.problem6(g)
        return g, 6, ego, prob
    prob, g, ego = tc.problem6(tc.small_graph(seed=11 if name == "6dof" else 13, n=40, loops=100), priors=name == "6dof_gravity")
    return g, 6, ego, prob


def well_conditioned(t):
    if t["kind"] not in (co.ACCEPTED, co.REJECTED, co.CONVERGED) or not np.isfinite(t["candidate_cost"]):
        return True
    return abs(t["relative_decrease"] - 1e-3) > 1e-6 and abs(t["cost"] - t["candidate_cost"]) > 1e-9 * t["cost"]


def close(a, b, rel=1e-10):
    if np.isnan(a) or np.isnan(b):
        return np.isnan(a) and np.isnan(b)
    return abs(a - b) <= rel * max(abs(a), abs(b), 1e-300)


def pose_bound(dof, x, y):
    dp, dr = tpa.pose_diff(dof, x, y) if dof == 4 else tc.pose_diff6(x, y)
    return dp, dr


def compare_traces(td, to, rep_d, rep_o):
    """step kinds equal and C, C+, m, radius within 1e-10 while the decisions are well conditioned; the termination when the
    oracle's last decision is; returns the iterations compared"""
    n = 0
    for k, t in enumerate(to):
        if not well_conditioned(t):
            return n
        assert k < len(td["kind"]), (k, len(td["kind"]))
        assert td["kind"][k] == t["kind"], (k, td["kind"][k], t)
        for f in ("cost", "candidate_cost", "model_cost_change", "radius"):
            assert close(td[f][k], t[f]), (k, f, td[f][k], t[f])
        n += 1
    assert len(td["kind"]) == len(to)
    assert (pgo.TERMINATIONS[rep_o["type"]], pgo.STOP_REASONS[rep_o["reason"]]) == (rep_d["termination"], rep_d["stop"])
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["6dof", "4dof", "6dof_gravity", "bench"])
def test_trace_matches_the_oracle(name):
    g, dof, ego, prob = case(name)
    cfg = dict(max_num_iterations=6) if name == "bench" else dict(function_tolerance=1e-12, max_num_iterations=60)
    x_o, to, rep_o = co.ceres_lm_solve(prob, **cfg)
    s = device(g, dof, ego, **cfg)
    r = s.solve()
    rep_d = s.minimizer_report(); td = s.debug_minimizer_trace(); x_d = poses(s, g, dof)
    s.close()
    assert compare_traces(td, to, rep_d, rep_o) >= 1
    assert r.iterations == rep_d["successful_steps"] + rep_d["unsuccessful_steps"] and r.accepted == rep_d["successful_steps"]
    assert r.converged == (rep_d["termination"] == "CONVERGENCE") and r.pcg_iterations == 0
    assert close(r.final_cost, rep_o["final_cost"]) and close(r.initial_cost, rep_o["initial_cost"])
    dp, dr = pose_bound(dof, x_d, x_o)
    assert dp < 1e-6 and dr < 1e-6, (dp, dr)


@pytest.mark.gpu
@pytest.mark.parametrize("dof", [4, 6])
def test_arock_local_solves_on_the_ceres_minimiser_match_the_oracle(dof):
    gg = tpa.graph(dof)
    cfg = tpa.SHIPPED["default"]
    lm = dict(max_num_iterations=100, function_tolerance=1e-10, parameter_tolerance=1e-12)
    dev = tpa.device_agents(gg, cfg, solver_kw=dict(linear_solver="sparse_cholesky"))
    for a in dev:
        a.s.set_minimizer("ceres_lm", **lm)
    orc = [co.arock_agent(pgo.arock_split(gg, k), lm, **cfg) for k in range(3)]
    for r in range(6):
        pgo.arock_run(dev, 1); ao.arock_run(orc, 1)
        for d, o in zip(dev, orc):
            dp, dr = tpa.pose_diff(dof, d.poses(), o.x)
            assert dp < 1e-6 and dr < 1e-6, (r, d.self_id, dp, dr)
            assert d.s.minimizer_report()["successful_steps"] >= 0
            dd = d.duals()
            assert sorted(dd) == sorted(o.duals)
            for key, (yl, yr) in dd.items():
                assert np.abs(yl - o.duals[key][0]).max() < 1e-6 and np.abs(yr - o.duals[key][1]).max() < 1e-6, (r, key)
    for a in dev:
        a.close()


@pytest.mark.gpu
def test_time_budget():
    g = tc.small_graph(seed=41, n=60, loops=150)
    s = device(g, 6, max_solver_time_in_seconds=1e-9)
    r = s.solve()
    rep = s.minimizer_report()
    assert r.iterations == 0 and rep["stop"] == "time" and rep["termination"] == "NO_CONVERGENCE"
    assert np.array_equal(s.get_poses(g["ids"]), np.asarray(g["init"], np.float64))
    s.close()
    free = dict(function_tolerance=0.0, parameter_tolerance=0.0, gradient_tolerance=0.0, max_num_iterations=100000)
    s = device(g, 6, max_solver_time_in_seconds=2e-3, **free)
    r = s.solve(); rep = s.minimizer_report(); xb = s.get_poses(g["ids"]); s.close()
    assert rep["stop"] == "time" and r.iterations > 0, rep
    free["max_num_iterations"] = r.iterations
    s = device(g, 6, **free)
    r2 = s.solve(); rep2 = s.minimizer_report(); xk = s.get_poses(g["ids"]); s.close()
    assert rep2["stop"] == "max_iterations" and r2.iterations == r.iterations
    assert np.array_equal(xb, xk)


@pytest.mark.gpu
def test_reproducible_and_one_synchronisation_per_solve():
    g = tc.with_extras(tc.small_graph(seed=31), repeat=5, selfs=3)
    runs = []
    for _ in range(2):
        s = device(g, 6)
        r = s.solve()
        runs.append((r.final_cost, s.get_poses(g["ids"]), s.debug_minimizer_trace(), s.minimizer_report()["host_syncs"]))
        r2 = s.solve()   # from the solved poses: the graph and the factor's tables are on the device already
        assert s.minimizer_report()["host_syncs"] == 1 and r2.final_cost <= r.final_cost
        s.close()
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1]) and runs[0][3] <= 3
    for k in runs[0][2]:
        assert np.array_equal(runs[0][2][k], runs[1][2][k], equal_nan=True), k


@pytest.mark.gpu
def test_refusals_keep_nothing():
    g = tc.small_graph(seed=51, n=30, loops=60)
    s = tc.device(g, 6, linear_solver="pcg")
    s.set_minimizer("ceres_lm")
    with pytest.raises(RuntimeError, match="rc=5"):
        s.solve()
    assert np.array_equal(s.get_poses(g["ids"]), np.asarray(g["init"], np.float64))
    with pytest.raises(RuntimeError, match="rc=5"):
        s.minimizer_report()
    for bad in (dict(function_tolerance=float("nan")), dict(initial_trust_region_radius=-1.0), dict(min_trust_region_radius=1e5),
                dict(min_lm_diagonal=1e3, max_lm_diagonal=1.0), dict(jacobi_scaling=2), dict(max_num_iterations=-1)):
        with pytest.raises(RuntimeError, match="rc=2"):
            s.set_minimizer("ceres_lm", **bad)
    with pytest.raises(ValueError):
        s.set_minimizer("dogleg")
    s.set_minimizer("restated")
    r = s.solve()
    assert r.iterations > 0
    with pytest.raises(RuntimeError, match="rc=5"):
        s.minimizer_report()
    s.close()
    # a refused config keeps the earlier one: the 1-iteration limit still holds
    s = device(g, 6, max_num_iterations=1)
    with pytest.raises(RuntimeError, match="rc=2"):
        s.set_minimizer("ceres_lm", parameter_tolerance=-1.0)
    assert s.solve().iterations == 1
    s.close()
    # ARock with the ceres minimiser on PCG: refused before the inbox or the duals change
    gg = tpa.graph(6)
    a = tpa.device_agents(gg, tpa.SHIPPED["default"], solver_kw=dict(linear_solver="pcg"))[0]
    a.s.set_minimizer("ceres_lm")
    before = a.duals()
    with pytest.raises(RuntimeError, match="rc=5"):
        a.step()
    assert a.duals() == before
    a.close()
